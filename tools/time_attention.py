"""Time the ViT attention forward / backward ops alone (CUDA events, qkv of 232 MB per call > L2).
python tools/time_attention.py [B] [T] [H]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from deeplearning_b200 import ops

B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
T = int(sys.argv[2]) if len(sys.argv) > 2 else 197
H = int(sys.argv[3]) if len(sys.argv) > 3 else 12
torch.manual_seed(0)
qkv = (torch.randn(B, T, 3 * H * 64, device="cuda") * 0.5).to(torch.bfloat16)
dout = (torch.randn(B, T, H * 64, device="cuda") * 0.1).to(torch.bfloat16)
scale = 64 ** -0.5


def timed(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


att, lse = ops.attention_fwd(qkv, H, scale)
# fp32 reference of the op on a slice of the batch
q, k, v = qkv[:4].float().view(4, T, 3, H, 64).permute(2, 0, 3, 1, 4)
ref = torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v
err = (att[:4].float().view(4, T, H, 64).permute(0, 2, 1, 3) - ref).abs().max().item()
t_f = timed(lambda: ops.attention_fwd(qkv, H, scale))
t_b = timed(lambda: ops.attention_bwd(qkv, att, dout, lse, H, scale))
fl = 4.0 * B * H * T * T * 64
print(f"attention B={B} T={T} H={H} : fwd {t_f:.1f} us ({fl / t_f / 1e6:.0f} TFLOP/s) "
      f"bwd(+delta) {t_b:.1f} us ({2.5 * fl / t_b / 1e6:.0f} TFLOP/s)  max|err| vs fp32 {err:.2e}")
