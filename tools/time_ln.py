"""Time LayerNorm backward alone at the shapes of the three transformer-style families (CUDA events; ops.Profiler spans so that
the finalize launch is not counted).
python tools/time_ln.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from deeplearning_b200 import ops

BF16, F32 = torch.bfloat16, torch.float32
CASES = [("ViT-B/16 bs256", 256 * 197, 768, F32, True), ("Swin-T s1 bs128", 128 * 3136, 96, F32, True),
         ("Swin-T s3 bs128", 128 * 196, 384, F32, True), ("ConvNeXt-T s1 bs256", 256 * 3136, 96, BF16, False),
         ("ConvNeXt-T s3 bs256", 256 * 196, 384, BF16, False)]
for name, rows, C, xdt, has_add in CASES:
    torch.manual_seed(0)
    x = torch.randn(rows, C, device="cuda", dtype=F32).to(xdt)
    dy = (torch.randn(rows, C, device="cuda") * 0.1).to(BF16)
    add = (torch.randn(rows, C, device="cuda") * 0.1).to(BF16) if has_add else None
    gamma = torch.rand(C, device="cuda") + 0.5
    y, mean, rstd = ops.layernorm_fwd(x, gamma, torch.zeros(C, device="cuda"), 1e-6)
    for _ in range(3):
        ops.layernorm_bwd(dy, x, mean, rstd, gamma, add=add)
    torch.cuda.synchronize()
    with ops.Profiler(run_ahead_ms=20.0) as prof:
        for _ in range(10):
            ops.layernorm_bwd(dy, x, mean, rstd, gamma, add=add)
    torch.cuda.synchronize()
    ts = [e0.elapsed_time(e1) * 1e3 for (n, fl, nb, e0, e1) in prof.records if n == "layernorm_bwd"]
    nbytes = x.numel() * x.element_size() + dy.numel() * 2 * (3 if has_add else 2)
    t = sorted(ts)[len(ts) // 2]
    print(f"layernorm_bwd {name:22s} rows {rows:7d} C {C:4d}: {t:7.1f} us  {nbytes / t / 1e6:6.2f} TB/s")
