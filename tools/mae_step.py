"""Throughput of MAE pre-training on the GPU engine, all in one invocation on one GPU: TrainStep graph img/s of train.py's
pre-training model (12 x 768 encoder, MLP 1024; 8 x 512 decoder, 16 heads of 64; mask ratio 0.75) with the recipe's AdamW
(betas 0.9 / 0.95, weight decay 0.05 on every parameter), and the fp32 oracle (oracle/mae.py) under bf16 autocast with the
same optimizer, with the FLOP rate of the step computed from shapes (about 58 GFLOP per image at 224 px).

    python tools/mae_step.py [--batch 256] [--steps 10] [--warmup 3] [--out FILE]

The first line names the card, its power limit and max SM clock, read in the same call."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.senet_step import _device_line, _timed  # noqa: E402

CFG = dict(image_size=224, patch_size=16, encoer_dim=768, mlp_dim=1024, encoder_depth=12, num_encoder_head=12,
           dim_per_head=64, decoder_dim=512, decoder_depth=8, num_decoder_head=16, mask_ratio=0.75)


def _model():
    from deeplearning_b200.self_supervised.MAE.models.MAE import MAEVisonTransformer

    torch.manual_seed(0)
    return MAEVisonTransformer(**CFG)


def _data(B):
    g = torch.Generator(device="cuda").manual_seed(1234)
    return torch.randn(B, 3, 224, 224, device="cuda", generator=g)


def step_gflop():
    """Forward + backward GFLOP per image (matmuls and attention; backward = 2x forward)."""
    P, Nm = 196, 147
    Nv = P - Nm
    K = 16 * 16 * 3

    def stack(T, D, inner, hidden, depth):
        return depth * (2 * T * D * 3 * inner + 4 * T * T * inner + 2 * T * inner * D + 4 * T * D * hidden)

    f = 2 * Nv * K * 768 + stack(Nv, 768, 768, 1024, 12) + 2 * Nv * 768 * 512 + stack(P, 512, 1024, 2048, 8) + 2 * Nm * 512 * K
    return 3 * f / 1e9


def engine_train(B, steps, warmup):
    from deeplearning_b200.engine.trainer import TrainStep

    model = _model().cuda().train()
    tr = TrainStep(model, lr=1.5e-4, optimizer="adamw", betas=(0.9, 0.95), weight_decay=0.05, no_decay=lambda n, p: False)
    x = _data(B)
    tr.step_eager(x)
    tr.capture(x)
    ms = _timed(lambda: tr.step(x), steps, warmup)
    del tr, model
    torch.cuda.empty_cache()
    return ms


def oracle_train(B, steps, warmup):
    from oracle.mae import mae_forward

    s = {k: v.cuda().requires_grad_() for k, v in _model().state_dict().items()}
    opt = torch.optim.AdamW(list(s.values()), lr=1.5e-4, betas=(0.9, 0.95), weight_decay=0.05)
    x = _data(B)
    P = 196

    def step():
        opt.zero_grad(set_to_none=True)
        shuffle = torch.rand(B, P, device="cuda").argsort()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            pred, target = mae_forward(s, x, shuffle, 16, 12, 16, 0.75)
        F.mse_loss(pred.float(), target).backward()
        opt.step()

    ms = _timed(step, steps, warmup)
    del s, opt
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mae_step.py measures on a CUDA device; none is available")
    B = a.batch
    gf = step_gflop()
    lines = [f"device: {_device_line()}"]
    ms = engine_train(B, a.steps, a.warmup)
    lines.append(f"pretrain MAE engine (graph, AdamW) bs {B} 224px: {ms:.1f} ms/step  {B * 1e3 / ms:.0f} img/s  "
                 f"{B * gf / ms:.0f} TFLOP/s ({gf:.1f} GFLOP/img)")
    ms = oracle_train(B, a.steps, a.warmup)
    lines.append(f"pretrain MAE oracle bf16 autocast bs {B}: {ms:.1f} ms/step  {B * 1e3 / ms:.0f} img/s")
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
