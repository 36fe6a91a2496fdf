"""Layer-by-layer error growth of the GPU ResNet-50 forward vs an fp32 PyTorch run, next to torch-autocast(bf16)'s own
error on the same weights/inputs (yardstick for what bf16 storage costs). python tools/debug_resnet_layers.py [B] [train|eval]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
import torchvision
from deeplearning_b200.classification.resnet.models.networks import resnet50
from deeplearning_b200.engine import resnet as engine

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
train = (sys.argv[2] if len(sys.argv) > 2 else "train") == "train"
torch.manual_seed(0)
m = resnet50().cuda()
ref = torchvision.models.resnet50().cuda()
ref.load_state_dict(m.state_dict())
m.train(train); ref.train(train)
x = torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

acts = {}
def hook(name):
    def f(mod, inp, out):
        acts[name] = out.detach().float()
    return f
names = []
for li in range(1, 5):
    for bi, blk in enumerate(getattr(ref, f"layer{li}")):
        n = f"layer{li}.{bi}"; names.append(n); blk.register_forward_hook(hook(n))
with torch.no_grad():
    ref_sd = {k: v.clone() for k, v in ref.state_dict().items()}
    logits_ref = ref(x).float()
    fp32_acts = dict(acts); acts.clear()
    ref.load_state_dict(ref_sd)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits_ac = ref(x).float()
    ac_acts = dict(acts)
    logits, tape = engine.forward(m, x, train, True)
for n, (units, ds, x_in) in zip(names, tape["blocks"]):
    mine = units[-1].y.float().permute(0, 3, 1, 2)
    r = fp32_acts[n]
    e_m = float((mine - r).norm() / r.norm()); e_a = float((ac_acts[n] - r).norm() / r.norm())
    print(f"{n:10s} rel-L2 err: b200 {e_m:.4f}   torch-autocast-bf16 {e_a:.4f}")
print(f"logits: |ref|max {float(logits_ref.abs().max()):.3f}  b200 max-abs err {float((logits - logits_ref).abs().max()):.4f}  "
      f"autocast max-abs err {float((logits_ac - logits_ref).abs().max()):.4f}")
