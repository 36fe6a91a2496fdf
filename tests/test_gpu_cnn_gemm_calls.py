"""Every GEMM call the CNN engines make, replayed against float64.

A module fixture wraps the GEMM entry points of ``deeplearning_b200.ops`` (``GEMM_OPS``) in recording shims and runs, for
every constructor in tests/test_cnn_admission.py (ResNet / ResNeXt / Wide-ResNet with ``B200_RESNET_ALGEBRA`` on and
off, SE-ResNet, VGG with and without BatchNorm, RepVGG, ShuffleNet v1 / v2, EfficientNet B0-B7) and MAE's pre-training
model: one batch-2 ``TrainStep`` at the native resolution, one eval forward, and for RepVGG one forward of the
re-parameterised model.  Only outermost calls are logged.  A call signature is the op, the shape and dtype of every tensor
argument, the integer options (ksize, stride, groups, act, in_hw, ...) and which optional arguments were given.

Each distinct signature is replayed once with fresh seeded inputs (batch 1 instead of 2 for images with more than one
pixel): bf16 activations, fp32 weights drawn in OIHW / [N][K] and packed by ``ops.pack_weight``, BatchNorm coefficients
of both signs whose ReLU masks are mixed and never within 0.05 of the boundary.  The float64 restatement is
``F.conv2d`` / ``torch.nn.grad.conv2d_input`` / ``conv2d_weight`` (with groups) plus the epilogue written out.  For every
signature: ``max|err| <= rel * max|ref|`` per output, bf16 outputs elementwise within ``2^-8 |ref| + K 2^-22 max|ref|``,
statistics rows against float64 sums of the stored output, padded columns exactly 0, and two launches bit-identical.
A recorded op without a replay fails the test.  A few signatures are also replayed at batch 256, where split-K and the
reduce slicing reach their largest counts.

Distinct replayed signatures (a signature shared by two families counts for both):
  conv2d_fwd 797 (efficientnet 369, repvgg 134, resnet 126, shufflenet_v1 107, shufflenet_v2 66, senet 58, vgg 21)
  conv2d_dgrad 475 (efficientnet 220, repvgg 88, resnet 83, shufflenet_v1 55, senet 35, shufflenet_v2 33, vgg 12)
  conv2d_wgrad 446 (efficientnet 188, repvgg 90, resnet 76, shufflenet_v1 56, shufflenet_v2 34, senet 30, vgg 12, mae 10)
  conv2d_bn_act 74 (resnet 66, vgg 9); gemm 22 (mae); im2col_nchw 9; gemm_dual 8 (resnet); conv1x1_bn_act 6;
  conv1x1_dgrad_masked 6; stem_wgrad_relayout 6; conv1x1_bn 2; stem_s2d_conv_fwd 2; stem_s2d_conv_wgrad 1;
  conv2d_fwd_f32 0 (ConvNeXt only).
The recording and every replay take about 30 s on an H100.

Every ``rel`` is at most 4x the largest ratio measured on an H100 80GB HBM3 (700 W), given in the comment beside it."""
import functools
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64

GEMM_OPS = ("conv2d_fwd", "conv2d_fwd_f32", "conv2d_bn_act", "conv2d_dgrad", "conv2d_wgrad", "gemm", "gemm_dual",
            "conv1x1_bn_act", "conv1x1_bn", "conv1x1_dgrad_masked", "stem_s2d_conv_fwd", "stem_s2d_conv_wgrad",
            "im2col_nchw", "stem_wgrad_relayout")
# image-shaped arguments of each op: these are replayed at batch 1
_IMAGE_ARGS = {"conv2d_fwd": ("x", "residual"), "conv2d_fwd_f32": ("x",), "conv2d_bn_act": ("x", "residual"),
               "conv2d_dgrad": ("dy", "residual", "out", "bn_mask"), "conv2d_wgrad": ("dy", "x"),
               "conv1x1_bn_act": ("x", "residual"), "conv1x1_bn": ("x",), "conv1x1_dgrad_masked": ("dy", "residual", "mask_src"),
               "stem_s2d_conv_fwd": ("z",), "stem_s2d_conv_wgrad": ("dy", "z"), "im2col_nchw": ("x",)}

# max|err| <= REL * max|ref| per (op, output); statistics: |err| <= REL * (float64 sum of |terms|) per column.  Every bf16
# output's worst ratio lies between 0.0024 and 0.0037 (one bf16 rounding at the largest value).
BF16_REL = 2 ** -7
REL = {
    ("conv2d_fwd", "y"): BF16_REL, ("conv2d_fwd", "y_f32"): 1e-5,         # 3.1e-6 (classifier head, K = 4096)
    ("conv2d_fwd", "stats"): 5e-7,                                         # 2.0e-7
    ("conv2d_bn_act", "y"): BF16_REL,
    ("conv2d_dgrad", "dx"): BF16_REL, ("conv2d_dgrad", "dz"): BF16_REL, ("conv2d_dgrad", "stats"): 1.5e-7,   # 4.4e-8
    ("conv2d_wgrad", "dw"): 5e-6,                                          # 1.5e-6
    ("conv2d_wgrad", "bias"): 1e-6,                                        # 2.6e-7
    ("gemm", "out"): BF16_REL, ("gemm", "out_f32"): 5e-6,                  # 1.7e-6
    ("gemm", "aux"): BF16_REL, ("gemm", "stats"): 5e-7,                    # 1.3e-7
    ("gemm_dual", "out"): BF16_REL, ("gemm_dual", "dz"): BF16_REL, ("gemm_dual", "stats"): 5e-8,   # 1.5e-8
    ("conv1x1_bn_act", "y"): BF16_REL, ("conv1x1_bn", "y"): BF16_REL,
    ("conv1x1_dgrad_masked", "dz"): BF16_REL, ("conv1x1_dgrad_masked", "stats"): 8e-9,   # 2.0e-9
    ("stem_s2d_conv_fwd", "y"): BF16_REL, ("stem_s2d_conv_fwd", "stats"): 1e-7,   # 2.7e-8
    ("stem_s2d_conv_wgrad", "dw"): 1e-6,                                   # 2.7e-7
}


# ------------------------------------------------------------------------------------------------------------ recording
def _desc(v):
    from deeplearning_b200 import ops

    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), str(v.dtype).split(".")[-1])
    if isinstance(v, ops.BnCoeffs):
        return ("co", v.scale.numel())
    if isinstance(v, (tuple, list)):
        return tuple(_desc(t) for t in v)
    return v


class Recording:
    def __init__(self):
        self.depth = 0
        self.sigs = {}        # (op, args) -> set of tags "family/constructor"
        self.outcome = {}     # (constructor, variant) -> ("train" | "reject" | "error", detail)
        self.tag = None

    def log(self, op, bound):
        args = {k: _desc(v) for k, v in bound.items()}
        if op == "conv2d_dgrad" and bound.get("out") is not None and bound["out"] is bound.get("residual"):
            args["out"] = "residual"
        self.sigs.setdefault((op, tuple(sorted(args.items()))), set()).add(self.tag)


def _shim(rec, op, fn):
    import inspect

    sig = inspect.signature(fn)

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        if rec.depth == 0:
            b = sig.bind(*args, **kwargs)
            b.apply_defaults()
            rec.log(op, b.arguments)
        rec.depth += 1
        try:
            return fn(*args, **kwargs)
        finally:
            rec.depth -= 1

    return wrapper


MAE_CFG = dict(image_size=224, patch_size=16, encoer_dim=768, mlp_dim=1024, encoder_depth=12, num_encoder_head=12,
               dim_per_head=64, decoder_dim=512, decoder_depth=8, num_decoder_head=16, mask_ratio=0.75)


def _runs():
    """(constructor name, variant, family, zero-argument constructor, resolution) of every recorded run."""
    import test_cnn_admission as adm

    out = []
    for name, (fam, fn, hw) in sorted(adm.CTORS.items()):
        for algebra in (("1", "0") if fam == "resnet" else (None,)):
            out.append((name, algebra, fam, fn, hw))

    def mae():
        from deeplearning_b200.self_supervised.MAE.models.MAE import MAEVisonTransformer

        return MAEVisonTransformer(**MAE_CFG)

    out.append(("mae_pretrain", None, "mae", mae, 224))
    return out


def _step(name, fam, fn, hw, expect):
    from deeplearning_b200 import ops
    from deeplearning_b200.engine.packing import weight_cache
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    with torch.device("cuda"):
        m = fn()
    x = torch.randn(2, 3, hw, hw, device="cuda")
    y = None if fam == "mae" else torch.tensor([3, 7], device="cuda")
    try:
        if expect == "reject":
            n0 = ops.launch_count()
            try:
                TrainStep(m).step_eager(x, y)
            except NotImplementedError as e:
                with torch.no_grad():
                    try:
                        m.eval()(x)
                    except NotImplementedError:
                        if ops.launch_count() == n0:
                            return ("reject", str(e))
                return ("error", f"launched {ops.launch_count() - n0} kernels before rejecting: {e}")
            return ("error", "not rejected")
        step = TrainStep(m)
        loss, _ = step.step_eager(x, y)
        torch.cuda.synchronize()
        if not bool(torch.isfinite(loss).all()) or not bool(torch.isfinite(step.arena.flat_g).all()):
            return ("error", "non-finite loss or gradient")
        m.eval()
        with torch.no_grad():
            out = m(x)
            outs = out if isinstance(out, tuple) else (out,)
            if fam == "repvgg":
                from deeplearning_b200.classification.RepVGG.models.repvgg import repvgg_model_convert

                outs += (repvgg_model_convert(m, do_copy=False)(x),)
        torch.cuda.synchronize()
        if not all(bool(torch.isfinite(o).all()) for o in outs):
            return ("error", "non-finite eval output")
        return ("train", f"loss {float(loss):.4f}")
    except Exception as e:   # recorded: a constructor that fails in the middle of a step is a finding
        return ("error", f"{type(e).__name__}: {e}")
    finally:
        del m
        weight_cache.clear()
        torch.cuda.empty_cache()


@functools.lru_cache(maxsize=None)
def recording():
    """Runs every constructor once per test session with the shims in place (shared with test_cnn_admission.py)."""
    import test_cnn_admission as adm
    from deeplearning_b200 import ops

    rec = Recording()
    saved = {op: getattr(ops, op) for op in GEMM_OPS}
    env = os.environ.get("B200_RESNET_ALGEBRA")
    try:
        for op in GEMM_OPS:
            setattr(ops, op, _shim(rec, op, saved[op]))
        for name, algebra, fam, fn, hw in _runs():
            if algebra is not None:
                os.environ["B200_RESNET_ALGEBRA"] = algebra
            rec.tag = f"{fam}/{name}"
            rec.outcome[(name, algebra)] = _step(name, fam, fn, hw, adm.EXPECT.get(name, "train"))
    finally:
        for op in GEMM_OPS:
            setattr(ops, op, saved[op])
        if env is None:
            os.environ.pop("B200_RESNET_ALGEBRA", None)
        else:
            os.environ["B200_RESNET_ALGEBRA"] = env
    return rec


def _batch1(op, args):
    """The replayed signature: image arguments of a batch-2 call with more than one pixel at batch 1."""
    img = _IMAGE_ARGS.get(op, ())

    def one(d):
        if isinstance(d, tuple) and len(d) == 3 and d[0] == "T" and len(d[1]) == 4 and d[1][0] == 2 and d[1][1] * d[1][2] > 1:
            return ("T", (1,) + d[1][1:], d[2])
        if isinstance(d, tuple) and d and isinstance(d[0], tuple):
            return tuple(one(t) for t in d)
        return d

    return tuple((k, one(v) if k in img else v) for k, v in args)


@functools.lru_cache(maxsize=None)
def replay_signatures():
    """{op: {replayed args: set of families}}"""
    rec = recording()
    out = {}
    for (op, args), tags in rec.sigs.items():
        out.setdefault(op, {}).setdefault(_batch1(op, args), set()).update(t.split("/")[0] for t in tags)
    return out


# ------------------------------------------------------------------------------------------------------------- inputs
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _act(shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=_gen(seed), device="cuda") * scale).to(BF16)


def _f32(shape, seed, scale=1.0):
    return torch.randn(*shape, generator=_gen(seed), device="cuda") * scale


def _weight(shape, seed):
    fan_in = 1
    for d in shape[1:]:
        fan_in *= d
    return _f32(shape, seed, 1.0 / math.sqrt(fan_in))


def _coeffs(C, seed):
    """BnCoeffs with scales of both signs (0.5 ... 1.5 in magnitude) and shifts of std 0.5"""
    from deeplearning_b200 import ops

    co = ops.BnCoeffs(C, "cuda")
    g = _gen(seed)
    mag = 0.5 + torch.rand(C, generator=g, device="cuda")
    sign = torch.where(torch.rand(C, generator=g, device="cuda") < 0.3, -1.0, 1.0)
    co.scale.copy_(mag * sign)
    co.shift.copy_(torch.randn(C, generator=g, device="cuda") * 0.5)
    co.mean.copy_(torch.randn(C, generator=g, device="cuda"))
    co.invstd.copy_(0.5 + torch.rand(C, generator=g, device="cuda"))
    return co


def _masked_raw(shape, co, seed):
    """x_raw bf16 whose BatchNorm + ReLU pre-activation u = x * scale + shift has mixed signs and |u| >= 0.05 everywhere,
    so that the fp32 mask of the kernel and the float64 mask of the reference agree"""
    g = _gen(seed)
    n = torch.randn(*shape, generator=g, device="cuda")
    u = torch.where(n >= 0, 1.0, -1.0) * (0.12 + n.abs())   # (randn can return exact zeros)
    x = ((u - co.shift) / co.scale).to(BF16)
    assert float((_d(x) * _d(co.scale) + _d(co.shift)).abs().min()) >= 0.05
    return x


def _d(t):
    return t.detach().double()


def _bf(w):
    """the bf16 rounding of an fp32 weight, in float64: what pack_weight hands the kernel"""
    return w.to(BF16).double()


def _nchw(t):
    return _d(t).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _pad(k):
    return 0 if k == 2 else k // 2


def _bn_alive(x_raw, co):
    return (_d(x_raw) * _d(co.scale) + _d(co.shift)) > 0


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# ------------------------------------------------------------------------------------------------------------- replays
class Unsupported(Exception):
    pass


def _T(a, name):
    d = a.get(name)
    return None if d is None else d


def _stats(got, cols):
    """float64 sums of a stats buffer [T, 2, C] over its rows (planes in `cols`)"""
    return _d(got).sum(0)[list(cols)]


def _replay(op, a, seed):
    """(launch, check): launch() runs the op on fresh inputs of signature `a` and returns its output tensors; check(outs)
    returns [(name, got, ref, kind, K)] with kind in bf16 / f32 / stats / exact and K the reduction length."""
    from deeplearning_b200 import ops

    a = dict(a)
    known = {"conv2d_fwd": _conv_fwd, "conv2d_fwd_f32": _conv_fwd, "conv2d_bn_act": _conv_fwd, "conv2d_dgrad": _conv_dgrad,
             "conv2d_wgrad": _conv_wgrad, "gemm": _gemm, "gemm_dual": _gemm_dual, "conv1x1_bn_act": _conv1x1,
             "conv1x1_bn": _conv1x1, "conv1x1_dgrad_masked": _conv1x1_dgrad_masked, "stem_s2d_conv_fwd": _stem_fwd,
             "stem_s2d_conv_wgrad": _stem_wgrad, "im2col_nchw": _im2col, "stem_wgrad_relayout": _relayout}
    if op not in known:
        raise Unsupported(f"no float64 reference for ops.{op}")
    return known[op](ops, op, a, seed)


def _conv_fwd(ops, op, a, seed):
    _, xs, _ = a["x"]
    B, H, W, Cin = xs
    k, s = a["ksize"], a["stride"]
    g = a.get("groups", 1)
    Cout, ld = a["w_packed"][1]
    if a.get("out_f32") and a.get("want_stats"):
        raise Unsupported("statistics of an fp32 output")
    x = _act(xs, seed)
    w = _weight((Cout, Cin // g, k, k), seed + 1)
    wp = ops.pack_weight(w, 3 if g != 1 else 0, ld=None if g != 1 else ld)
    if tuple(wp.shape) != (Cout, ld):
        raise Unsupported(f"packed operand {tuple(wp.shape)} != recorded {(Cout, ld)}")
    bias = _f32((Cout,), seed + 2) if a.get("bias") is not None else None
    res = _act(a["residual"][1], seed + 3) if a.get("residual") is not None else None
    co = _coeffs(Cout, seed + 4) if op == "conv2d_bn_act" else None

    def launch():
        if op == "conv2d_fwd":
            y, st = ops.conv2d_fwd(x, wp, k, s, want_stats=a["want_stats"], bias=bias, act=a["act"], residual=res,
                                   out_f32=a["out_f32"], groups=g)
            return (y,) if st is None else (y, st)
        if op == "conv2d_fwd_f32":
            return (ops.conv2d_fwd_f32(x, wp, k, s, bias=bias),)
        return (ops.conv2d_bn_act(x, wp, co, k, s, relu=a["relu"], residual=res, groups=g),)

    def check(outs):
        ref = _nhwc(F.conv2d(_nchw(x), _bf(w), stride=s, padding=_pad(k), groups=g))
        if op == "conv2d_bn_act":
            ref = ref * _d(co.scale) + _d(co.shift)
            if res is not None:
                ref = ref + _d(res)
            if a["relu"]:
                ref = ref.clamp_min(0)
        else:
            if bias is not None:
                ref = ref + _d(bias)
            if a.get("act", 0) == 1:
                ref = ref.clamp_min(0)
            elif a.get("act", 0) != 0:
                raise Unsupported(f"act {a['act']}")
            if res is not None:
                ref = ref + _d(res)
        y = outs[0]
        K = Cin // g * k * k
        r = [("y", y, ref, "f32" if y.dtype == F32 else "bf16", K)]
        if len(outs) > 1:
            yd = _d(y).reshape(-1, Cout)
            r.append(("stats", _stats(outs[1], (0, 1)), torch.stack([yd.sum(0), (yd * yd).sum(0)]), "stats",
                      torch.stack([yd.abs().sum(0), (yd * yd).sum(0)])))
        return r

    return launch, check


def _conv_dgrad(ops, op, a, seed):
    B, Ho, Wo, Cout = a["dy"][1]
    H, W = a["in_hw"]
    k, s = a["ksize"], a["stride"]
    g = a.get("groups", 1)
    Cin, ld = a["wd_packed"][1]
    dy = _act((B, Ho, Wo, Cout), seed)
    w = _weight((Cout, Cin // g, k, k), seed + 1)
    wd = ops.pack_weight(w, 4 if g != 1 else 1, ld=None if g != 1 else ld)
    if tuple(wd.shape) != (Cin, ld):
        raise Unsupported(f"packed operand {tuple(wd.shape)} != recorded {(Cin, ld)}")
    res = _act((B, H, W, Cin), seed + 2) if a.get("residual") is not None else None
    out0 = None
    if a.get("out") not in (None, "residual"):
        out0 = _act((B, H, W, Cin), seed + 3)
    mask = None
    if a.get("bn_mask") is not None:
        co = _coeffs(Cin, seed + 4)
        mask = (_masked_raw((B, H, W, Cin), co, seed + 5), co)

    def launch():
        r = None if res is None else res.clone()
        out = r if a.get("out") == "residual" else (None if out0 is None else out0.clone())
        o = ops.conv2d_dgrad(dy, wd, (H, W), k, s, residual=r, out=out, bn_mask=mask, groups=g)
        return o if isinstance(o, tuple) else (o,)

    def check(outs):
        ref = _nhwc(torch.nn.grad.conv2d_input((B, Cin, H, W), _bf(w), _nchw(dy), stride=s, padding=_pad(k), groups=g))
        if out0 is not None:
            if k == 1 and s == 2:   # only the even pixels are written
                keep = torch.ones(B, H, W, 1, dtype=torch.bool, device="cuda")
                keep[:, ::2, ::2] = False
                ref = torch.where(keep, _d(out0), ref)
        if res is not None:
            ref = ref + _d(res)
        K = Cout // g * k * k
        if mask is None:
            return [("dx", outs[0], ref, "bf16", K)]
        x_raw, _ = mask
        ref = torch.where(_bn_alive(x_raw, mask[1]), ref, torch.zeros_like(ref))
        dz = _d(outs[0]).reshape(-1, Cin)
        xr = _d(x_raw).reshape(-1, Cin)
        sref = torch.stack([dz.sum(0), (dz * xr).sum(0)])
        return [("dz", outs[0], ref, "bf16", K), ("stats", _stats(outs[1], (0, 1)), sref, "stats",
                                                  torch.stack([dz.abs().sum(0), (dz * xr).abs().sum(0)]))]

    return launch, check


def _wgrad_ref(x, dy, k, s, g, Cout):
    Cin = x.shape[-1]
    return torch.nn.grad.conv2d_weight(_nchw(x), (Cout, Cin // g, k, k), _nchw(dy), stride=s, padding=_pad(k), groups=g)


def _conv_wgrad(ops, op, a, seed):
    dys, xs = a["dy"][1], a["x"][1]
    k, s = a["ksize"], a["stride"]
    g = a.get("groups", 1)
    Cout = dys[-1]
    dy = _act(dys, seed)
    x = _act(xs, seed + 1)
    out0 = _f32(a["out"][1], seed + 2) if a.get("out") is not None else None
    gb = a.get("bias_out") is not None

    def launch():
        out = None if out0 is None else out0.clone()
        bo = torch.full((Cout,), float("nan"), device="cuda") if gb else None
        dw = ops.conv2d_wgrad(dy, x, k, s, out=out, accumulate=a["accumulate"], bias_out=bo, groups=g)
        return (dw,) if bo is None else (dw, bo)

    def check(outs):
        ref = _wgrad_ref(x, dy, k, s, g, Cout).reshape(outs[0].shape)
        if out0 is not None and a["accumulate"]:
            ref = ref + _d(out0)
        r = [("dw", outs[0], ref, "f32", None)]
        if gb:
            r.append(("bias", outs[1], _d(dy).reshape(-1, Cout).sum(0), "f32", None))
        return r

    return launch, check


def _gemm(ops, op, a, seed):
    for opt in ("out", "a_view", "out_view", "residual_view"):
        if a.get(opt) is not None:
            raise Unsupported(f"gemm with {opt}=")
    if a.get("out_offset", 0) != 0:
        raise Unsupported("gemm with out_offset")
    N, K = a["w_packed"][1]
    x = _act(a["a"][1], seed)
    rows = x.numel() // K
    w = _weight((N, K), seed + 1)
    wp = ops.pack_weight(w, 0)
    bias = _f32((N,), seed + 2) if a.get("bias") is not None else None
    res = None
    if a.get("residual") is not None:
        _, rs, rdt = a["residual"]
        res = _act(rs, seed + 3) if rdt == "bfloat16" else _f32(rs, seed + 3)
    aux_in = None
    if a.get("aux_in") is not None:
        aux_in = (torch.rand(*a["aux_in"][1], generator=_gen(seed + 4), device="cuda") * 1.2 - 0.1).to(BF16)
    colscale = _f32((N,), seed + 5) if a.get("colscale") is not None else None
    rowscale = None
    if a.get("rowscale") is not None:
        (_, (S,), _), rps = a["rowscale"]
        rowscale = ((torch.rand(S, generator=_gen(seed + 6), device="cuda") < 0.7).float() * 1.25, rps)
    act = a.get("act", 0)

    def launch():
        r = ops.gemm(x, wp, bias=bias, act=act, out_f32=a["out_f32"], residual=res, aux_out=a["aux_out"], aux_in=aux_in,
                     want_stats=a["want_stats"], colscale=colscale, rowscale=rowscale)
        return tuple(t for t in r if t is not None)

    def check(outs):
        pre = _d(x).reshape(rows, K) @ _bf(w).T
        if bias is not None:
            pre = pre + _d(bias)
        aux = _gelu_grad(pre) if act == 2 else pre
        post = {0: pre, 1: pre.clamp_min(0), 2: _gelu(pre)}.get(act)
        if act == 3:
            post = pre * _d(aux_in).reshape(rows, N)
        if colscale is not None:
            post = post * _d(colscale)
        if rowscale is not None:
            post = post * _d(rowscale[0]).repeat_interleave(rowscale[1])[:rows, None]
        if res is not None:
            post = post + _d(res).reshape(rows, N)
        y = outs[0]
        r = [("out", y, post.reshape(y.shape), "f32" if y.dtype == F32 else "bf16", K)]
        i = 1
        if a["aux_out"]:
            r.append(("aux", outs[1], aux.reshape(outs[1].shape), "bf16", K))
            i = 2
        if a["want_stats"]:
            yd = _d(y).reshape(rows, N)
            r.append(("stats", _stats(outs[i], (0, 1)), torch.stack([yd.sum(0), (yd * yd).sum(0)]), "stats",
                      torch.stack([yd.abs().sum(0), (yd * yd).sum(0)])))
        return r

    return launch, check


def _gemm_dual(ops, op, a, seed):
    s0, s1 = a["a0"][1], a["a1"][1]
    K0, K1 = s0[-1], s1[-1]
    N = a["wcat"][1][0]
    a0, a1 = _act(s0, seed), _act(s1, seed + 1)
    w = _weight((N, K0 + K1), seed + 2)
    wcat = ops.pack_weight(w, 0)
    bias = _f32((N,), seed + 3)
    mask = None
    if a.get("bn_mask") is not None:
        co = _coeffs(N, seed + 4)
        mask = (_masked_raw(a["bn_mask"][0][1], co, seed + 5), co)

    def launch():
        o = ops.gemm_dual(a0, a1, wcat, bias, bn_mask=mask)
        return o if isinstance(o, tuple) else (o,)

    def check(outs):
        rows = a0.numel() // K0
        ref = torch.cat([_d(a0).reshape(rows, K0), _d(a1).reshape(rows, K1)], 1) @ _bf(w).T + _d(bias)
        if mask is None:
            return [("out", outs[0], ref.reshape(outs[0].shape), "bf16", K0 + K1)]
        alive = _bn_alive(mask[0], mask[1]).reshape(rows, N)
        ref = torch.where(alive, ref, torch.zeros_like(ref))
        dz = _d(outs[0]).reshape(rows, N)
        xr = _d(mask[0]).reshape(rows, N)
        return [("dz", outs[0], ref.reshape(outs[0].shape), "bf16", K0 + K1),
                ("stats", _stats(outs[1], (0, 1)), torch.stack([dz.sum(0), (dz * xr).sum(0)]), "stats",
                 torch.stack([dz.abs().sum(0), (dz * xr).abs().sum(0)]))]

    return launch, check


def _conv1x1(ops, op, a, seed):
    xs = a["x"][1]
    Cin = xs[-1]
    Cout = a["w_packed"][1][0]
    x = _act(xs, seed)
    w = _weight((Cout, Cin), seed + 1)
    wp = ops.pack_weight(w, 0)
    co = _coeffs(Cout, seed + 2)
    res = _act(a["residual"][1], seed + 3) if op == "conv1x1_bn_act" else None

    def launch():
        return (ops.conv1x1_bn_act(x, wp, co, res),) if res is not None else (ops.conv1x1_bn(x, wp, co),)

    def check(outs):
        ref = (_d(x).reshape(-1, Cin) @ _bf(w).T) * _d(co.scale) + _d(co.shift)
        if res is not None:
            ref = (ref + _d(res).reshape(-1, Cout)).clamp_min(0)
        return [("y", outs[0], ref.reshape(outs[0].shape), "bf16", Cin)]

    return launch, check


def _conv1x1_dgrad_masked(ops, op, a, seed):
    dys = a["dy"][1]
    Cout = dys[-1]
    Cin = a["wd_packed"][1][0]
    dy = _act(dys, seed)
    w = _weight((Cout, Cin), seed + 1)
    wd = ops.pack_weight(w, 1)
    res = _act(a["residual"][1], seed + 2)
    mask_src = _act(a["mask_src"][1], seed + 3).clamp_min(0)   # a ReLU output: about half exact zeros

    def launch():
        return ops.conv1x1_dgrad_masked(dy, wd, res, mask_src)

    def check(outs):
        ref = _d(dy).reshape(-1, Cout) @ _bf(w) + _d(res).reshape(-1, Cin)
        ref = torch.where(_d(mask_src).reshape(-1, Cin) > 0, ref, torch.zeros_like(ref))
        dz = _d(outs[0]).reshape(-1, Cin)
        return [("dz", outs[0], ref.reshape(outs[0].shape), "bf16", Cout),
                ("stats", _stats(outs[1], (0,)), dz.sum(0, keepdim=True), "stats", dz.abs().sum(0, keepdim=True))]

    return launch, check


def _stem_input(zs, seed):
    from deeplearning_b200 import ops

    B, Hz, Wz, _ = zs
    x = _f32((B, 3, 2 * (Hz - 3), 2 * (Wz - 3)), seed)
    z = ops.stem_s2d(x)
    assert tuple(z.shape) == tuple(zs)
    return x, z


def _stem_fwd(ops, op, a, seed):
    x, z = _stem_input(a["z"][1], seed)
    from deeplearning_b200.engine.packing import ModelPack

    w = _weight((64, 3, 7, 7), seed + 1)
    pk = ModelPack([(w, 2, 256, 64, (64, 3, 49))])   # the space-to-depth operand (mode 2) only comes from the pack table
    pk.refresh(0)
    wp = pk.get(w, 2)
    if tuple(wp.shape) != tuple(a["w_packed"][1]):
        raise Unsupported(f"stem operand {tuple(wp.shape)} != recorded {a['w_packed'][1]}")

    def launch():
        y, st = ops.stem_s2d_conv_fwd(z, wp, want_stats=a["want_stats"])
        return (y,) if st is None else (y, st)

    def check(outs):
        ref = _nhwc(F.conv2d(_bf(x), _bf(w), stride=2, padding=3))
        r = [("y", outs[0], ref, "bf16", 147)]
        if len(outs) > 1:
            yd = _d(outs[0]).reshape(-1, 64)
            r.append(("stats", _stats(outs[1], (0, 1)), torch.stack([yd.sum(0), (yd * yd).sum(0)]), "stats",
                      torch.stack([yd.abs().sum(0), (yd * yd).sum(0)])))
        return r

    return launch, check


def _stem_wgrad(ops, op, a, seed):
    x, z = _stem_input(a["z"][1], seed)
    dy = _act(a["dy"][1], seed + 1)
    out0 = _f32((64, 3, 7, 7), seed + 2) if a.get("out") is not None else None

    def launch():
        out = None if out0 is None else out0.clone()
        return (ops.stem_s2d_conv_wgrad(dy, z, out=out, accumulate=a["accumulate"]),)

    def check(outs):
        ref = torch.nn.grad.conv2d_weight(_bf(x), (64, 3, 7, 7), _nchw(dy), stride=2, padding=3)
        if out0 is not None and a["accumulate"]:
            ref = ref + _d(out0)
        return [("dw", outs[0], ref, "f32", None)]

    return launch, check


def _im2col(ops, op, a, seed):
    xs = a["x"][1]
    KH, KW, s, p, ldk = a["KH"], a["KW"], a["stride"], a["pad"], a["ldk"]
    x = _f32(xs, seed)

    def launch():
        return (ops.im2col_nchw(x, KH, KW, s, p, ldk)[0],)

    def check(outs):
        B, C = xs[0], xs[1]
        u = F.unfold(_bf(x), (KH, KW), padding=p, stride=s)            # [B, C*KH*KW, L], row = c*KH*KW + tap
        L = u.shape[-1]
        u = u.view(B, C, KH * KW, L).permute(0, 3, 2, 1).reshape(B * L, KH * KW * C)
        ref = torch.zeros(B * L, ldk, dtype=F64, device="cuda")
        ref[:, :KH * KW * C] = u
        return [("a", outs[0], ref, "exact", None)]

    return launch, check


def _relayout(ops, op, a, seed):
    cout, cin, taps = a["cout"], a["cin"], a["taps"]
    src = _f32(a["src"][1], seed)
    out0 = _f32(a["out"][1], seed + 1) if a.get("out") is not None else None
    k = int(round(taps ** 0.5))

    def launch():
        out = None if out0 is None else out0.clone()
        return (ops.stem_wgrad_relayout(src, cout, cin, taps, out=out, accumulate=a["accumulate"]),)

    def check(outs):
        ref = src[:, :taps * cin].reshape(cout, taps, cin).permute(0, 2, 1).reshape(cout, cin, k, k)
        if out0 is not None and a["accumulate"]:
            ref = out0 + ref   # fp32, as the kernel adds
        return [("dw", outs[0], ref, "exact", None)]

    return launch, check


# ------------------------------------------------------------------------------------------------------------- checking
def _compare(op, name, got, ref, kind, K):
    """[] or a list of failure strings; prints the measured ratio"""
    if tuple(got.shape) != tuple(ref.shape):
        return [f"{name}: shape {tuple(got.shape)} != {tuple(ref.shape)}"]
    if kind == "exact":
        ok = torch.equal(got, ref.to(got.dtype)) if got.dtype != F64 else torch.equal(got, ref)
        return [] if ok else [f"{name}: not exact ({float((_d(got) - _d(ref)).abs().max()):.3g})"]
    g, r = _d(got), _d(ref)
    fails = []
    if not bool(torch.isfinite(g).all()):
        return [f"{name}: non-finite output"]
    err = (g - r).abs()
    key = (op, name + ("_f32" if kind == "f32" and got.dtype == F32 and op in ("conv2d_fwd", "conv2d_fwd_f32", "gemm") else ""))
    if key not in REL:
        return [f"{name}: no tolerance for {key}"]
    rel = REL[key]
    if kind == "stats":
        # per column: fp32 partial sums of the stored values, bounded by their absolute sums
        ratio = float((err / (K + 1e-30)).max())
        if bool((err > K * rel).any()):
            fails.append(f"{name}: stats err / sum|.| = {ratio:.3g} > {rel:.3g}")
        return fails, ratio
    scale = float(r.abs().max())
    ratio = float(err.max()) / max(scale, 1e-30)
    if ratio > rel:
        fails.append(f"{name}: max err / max|ref| = {ratio:.3g} > {rel:.3g}")
    if kind == "bf16":
        bound = 2.0 ** -8 * r.abs() + K * 2.0 ** -22 * scale
        over = err > bound
        if bool(over.any()):
            i = int(over.flatten().nonzero()[0])
            fails.append(f"{name}: {int(over.sum())} elements beyond 2^-8|ref| + K 2^-22 max|ref| (first: got "
                         f"{float(g.flatten()[i]):.6g}, ref {float(r.flatten()[i]):.6g})")
    return fails, ratio


def run_signature(op, args, seed=1):
    """(failures, {output: ratio}) of one replayed signature"""
    launch, check = _replay(op, args, seed)
    o1 = launch()
    o2 = launch()
    torch.cuda.synchronize()
    fails, ratios = [], {}
    for i, (t1, t2) in enumerate(zip(o1, o2)):
        if not torch.equal(t1, t2):
            fails.append(f"output {i}: two launches differ")
    for name, got, ref, kind, K in check(o1):
        res = _compare(op, name, got, ref, kind, K)
        if isinstance(res, list):
            fails += res
            continue
        f, ratios[f"{name}:{kind}"] = res
        fails += f
    return fails, ratios


def _fmt(args):
    return ", ".join(f"{k}={v[1] if isinstance(v, tuple) and v and v[0] == 'T' else v}" for k, v in args
                     if v is not None and v is not False)


# ------------------------------------------------------------------------------------------------------------- tests
def test_recorded_ops_have_references():
    sigs = replay_signatures()
    unknown = sorted(op for op in sigs if op not in GEMM_OPS)
    assert not unknown
    for op, table in sorted(sigs.items()):
        fams = {}
        for args, fs in table.items():
            for f in fs:
                fams[f] = fams.get(f, 0) + 1
        print(f"{op}: {len(table)} signatures; per family {dict(sorted(fams.items()))}")
    assert sum(len(t) for t in sigs.values()) > 0


@pytest.mark.parametrize("op", GEMM_OPS)
def test_replay_against_float64(op):
    table = replay_signatures().get(op, {})
    failures, worst = [], {}
    for n, args in enumerate(sorted(table, key=repr)):
        try:
            fails, ratios = run_signature(op, args, seed=1 + 17 * n)
        except Unsupported as e:
            fails, ratios = [f"no reference: {e}"], {}
        for k, v in ratios.items():
            if v > worst.get(k, (-1.0, None))[0]:
                worst[k] = (v, args)
        if fails:
            failures.append(f"{op}({_fmt(args)}) [{','.join(sorted(table[args]))}]: " + "; ".join(fails))
    for k, (v, args) in sorted(worst.items()):
        print(f"{op} {k}: worst ratio {v:.3g} at {_fmt(args)}")
    print(f"{op}: {len(table)} signatures, {len(failures)} failing")
    assert not failures, "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------------ production scale
PROD_B = 256
# (what, recorded batch-1 signature it scales up: (dy shape, x shape, ksize, bias gradient), family)
PROD_WGRAD = {
    "vgg_conv0": (((1, 224, 224, 64), (1, 224, 224, 32), 1, True), "vgg"),                 # the K = 32 im2col GEMM
    "resnet_layer1_3x3": (((1, 56, 56, 64), (1, 56, 56, 64), 3, False), "resnet"),         # merged-tap tiles
    "efficientnet_b0_expand_1152": (((1, 7, 7, 1152), (1, 7, 7, 192), 1, False), "efficientnet"),
}
# (dw, bias) rel; measured dw 1.2e-4 / bias 3.3e-7, 1.9e-5, 9.6e-7 (fp32 split-K partials over 12.8 M / 803 k / 12.5 k rows)
PROD_REL = {"vgg_conv0": (4e-4, 1e-6), "resnet_layer1_3x3": (6e-5, None), "efficientnet_b0_expand_1152": (3e-6, None)}


def _wgrad_f64(dy, x, k, chunk=32):
    """float64 dw [Cout, Cin, k, k] of a stride-1 convolution, tap by tap and in batch chunks (on the GPU)"""
    B, H, W, Cin = x.shape
    Cout, p = dy.shape[-1], k // 2
    dw = torch.zeros(Cout, Cin, k, k, dtype=F64, device="cuda")
    for b0 in range(0, B, chunk):
        xp = F.pad(_d(x[b0:b0 + chunk]), (0, 0, p, p, p, p))
        dyf = _d(dy[b0:b0 + chunk]).reshape(-1, Cout)
        for kh in range(k):
            for kw in range(k):
                dw[:, :, kh, kw] += dyf.T @ xp[:, kh:kh + H, kw:kw + W].reshape(-1, Cin)
    return dw


@pytest.mark.parametrize("what", sorted(PROD_WGRAD))
def test_wgrad_at_batch_256(what):
    from deeplearning_b200 import ops

    (dys, xs, k, with_bias), fam = PROD_WGRAD[what]
    recorded = [a for a, fams in replay_signatures().get("conv2d_wgrad", {}).items()
                if fam in fams and dict(a)["dy"][1] == dys and dict(a)["x"][1] == xs and dict(a)["ksize"] == k
                and (dict(a)["bias_out"] is not None) == with_bias]
    assert recorded, f"{what}: the engine no longer makes this call"
    dy = _act((PROD_B,) + dys[1:], 11)
    x = _act((PROD_B,) + xs[1:], 12)
    pad_cols = 27 if what == "vgg_conv0" else xs[-1]
    if pad_cols < xs[-1]:
        x[..., pad_cols:] = 0          # the zero columns of the 3x3x3 patch matrix
    outs = []
    for _ in range(2):
        bo = torch.full((dys[-1],), float("nan"), device="cuda") if with_bias else None
        outs.append((ops.conv2d_wgrad(dy, x, k, 1, bias_out=bo), bo))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and (not with_bias or torch.equal(outs[0][1], outs[1][1]))
    dw, bo = outs[0]
    ref = _wgrad_f64(dy, x, k)
    ratio = float((_d(dw) - ref).abs().max() / ref.abs().max())
    print(f"{what}: dw max err / max|ref| = {ratio:.3g}")
    assert ratio <= PROD_REL[what][0]
    assert torch.equal(dw[:, pad_cols:], torch.zeros_like(dw[:, pad_cols:])), "padded columns of dw are not 0"
    if with_bias:
        bref = _d(dy).reshape(-1, dys[-1]).sum(0)
        ratio = float((_d(bo) - bref).abs().max() / bref.abs().max())
        print(f"{what}: bias max err / max|ref| = {ratio:.3g}")
        assert ratio <= PROD_REL[what][1]


def test_efficientnet_1152_fwd_dgrad_at_batch_256():
    """the 192 -> 1152 expand convolution of EfficientNet-B0 at batch 256: forward with statistics and the data gradient"""
    from deeplearning_b200 import ops

    for op, a in (("conv2d_fwd", dict(x=("T", (PROD_B, 7, 7, 192), "bfloat16"), w_packed=("T", (1152, 192), "bfloat16"),
                                      ksize=1, stride=1, want_stats=True, bias=None, act=0, residual=None, out_f32=False,
                                      groups=1)),
                  ("conv2d_dgrad", dict(dy=("T", (PROD_B, 7, 7, 1152), "bfloat16"), wd_packed=("T", (192, 1152), "bfloat16"),
                                        in_hw=(7, 7), ksize=1, stride=1, residual=None, out=None, bn_mask=None, groups=1))):
        recorded = replay_signatures().get(op, {})
        one = tuple(sorted((k, ("T", (1,) + v[1][1:], v[2]) if k in ("x", "dy") else v) for k, v in a.items()))
        assert one in recorded, f"{op}: the engine no longer makes this call"
        fails, ratios = run_signature(op, tuple(sorted(a.items())), seed=21)
        print(op, ratios)
        assert not fails, fails
