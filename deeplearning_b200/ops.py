"""Tensor-level wrappers over the C ABI (include/b200cls.h).

PyTorch is used for device memory and streams only; every arithmetic op below is a hand-written sm_90a kernel.
Activations are NHWC bf16 tensors ``[B, H, W, C]`` (``[rows, C]`` for linear layers); parameters and statistics fp32.
"""
import torch

from . import _lib

BF16 = torch.bfloat16
F32 = torch.float32


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _call(sym, *args):
    """Launch entry b200_<sym>(*args, stream) on the current stream; raises RuntimeError with the library's message."""
    rc = getattr(_lib.load(), "b200_" + sym)(*args, _stream())
    if rc:
        _lib.check(rc, "b200_" + sym)


# size_t sizing entries whose 0 result means an unsupported shape (include/b200cls.h); the int ones fail with -1
_ZERO_FAILS = frozenset({"conv2d_grouped_wgrad_workspace_bytes"})


def _query(sym, *args):
    """Value of the sizing entry b200_<sym>(*args) (rows, blocks, slices, splits, bytes); raises RuntimeError on the entry's
    failure value."""
    v = getattr(_lib.load(), "b200_" + sym)(*args)
    if (v == 0) if sym in _ZERO_FAILS else (v < 0):
        raise RuntimeError(f"b200_{sym}{args} failed: {_lib.last_error()}")
    return v


# ---------------------------------------------------------------------------------------------------- op-level profiler
_active_prof = None


class Profiler:
    """Times every C-ABI op with CUDA events on the launching stream and attributes algorithmic flops / bytes to it.
    Used by bench.py (roofline numbers) and tools/; zero cost when not active."""

    def __init__(self, run_ahead_ms=0.0):
        """run_ahead_ms > 0: park the stream on a spin kernel for about that long first, so the host enqueues the profiled
        region ahead of the device and the event spans measure kernel time, not host launch gaps."""
        self.records = []  # (name, flops, bytes, ev0, ev1)
        self.run_ahead_ms = run_ahead_ms

    def __enter__(self):
        global _active_prof
        self._prev, _active_prof = _active_prof, self
        if self.run_ahead_ms > 0:
            torch.cuda._sleep(int(self.run_ahead_ms * 1.9e6))  # cycles at ~1.9 GHz
        return self

    def __exit__(self, *exc):
        global _active_prof
        _active_prof = self._prev

    def summary(self):
        torch.cuda.synchronize()
        agg = {}
        for name, flops, nbytes, e0, e1 in self.records:
            a = agg.setdefault(name, {"calls": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            a["calls"] += 1
            a["ms"] += e0.elapsed_time(e1)
            a["flops"] += flops
            a["bytes"] += nbytes
        return agg


class _Span:
    __slots__ = ("name", "flops", "nbytes", "e0")

    def __init__(self, name, flops, nbytes):
        self.name, self.flops, self.nbytes = name, flops, nbytes

    def __enter__(self):
        self.e0 = torch.cuda.Event(enable_timing=True)
        self.e0.record()

    def __exit__(self, *exc):
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        _active_prof.records.append((self.name, self.flops, self.nbytes, self.e0, e1))


class _NoSpan:
    __slots__ = ()

    def __enter__(self):
        pass

    def __exit__(self, *exc):
        pass


_NO_SPAN = _NoSpan()


def _span(name, flops=0.0, *tensors):
    """``with _span(name, flops, *tensors):`` around an op's launches records it in the active Profiler, with the bytes of
    ``tensors`` (None entries skipped) as its traffic.  Without a Profiler it does nothing and counts no bytes."""
    return _NO_SPAN if _active_prof is None else _Span(name, flops, _nb(*tensors))


def _nb(*ts):
    return float(sum(t.numel() * t.element_size() for t in ts if t is not None))


def _chk_act(t, name):
    if t.dtype != BF16 or not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name}: expected a contiguous CUDA bf16 tensor, got {t.dtype} {t.device} contiguous={t.is_contiguous()}")


def out_hw(h, ksize, stride):
    pad = 0 if ksize == 2 else ksize // 2
    return (h + 2 * pad - ksize) // stride + 1


# --------------------------------------------------------------------------------------------------------- packing
def pack_weight(w, mode=0, ld=None):
    """fp32 OIHW (or [out,in]) parameter -> bf16 GEMM operand. mode 0: [O][taps*I]; mode 1 (dgrad): [I][taps*O];
    modes 3 / 4: block-diagonal forward / dgrad operands [C][taps*64] of a grouped convolution weight [C][C/groups][k][k]."""
    w = w.detach()
    if w.dtype != F32 or not w.is_contiguous():
        w = w.float().contiguous()
    O, I = w.shape[0], w.shape[1]
    taps = 1
    for d in w.shape[2:]:
        taps *= d
    rows = I if mode == 1 else O
    cols = taps * {0: I, 1: O}.get(mode, 64)
    ld = cols if ld is None else ld
    out = torch.empty(rows, ld, dtype=BF16, device=w.device)
    _call("pack_weight", _p(w), _p(out), O, I, taps, mode, ld)
    return out


def cast_bf16(x):
    x = x.contiguous()
    out = torch.empty(x.shape, dtype=BF16, device=x.device)
    _call("cast_f32_to_bf16", _p(x), _p(out), x.numel())
    return out


def cast_f32(x):
    out = torch.empty(x.shape, dtype=F32, device=x.device)
    _call("cast_bf16_to_f32", _p(x), _p(out), x.numel())
    return out


def im2col_nchw(x, KH, KW, stride, pad, ldk):
    """Stem only: fp32 NCHW batch -> bf16 [B*Ho*Wo, ldk] patch matrix (k = (kh*KW+kw)*Cin + c)."""
    B, C, H, W = x.shape
    Ho = (H + 2 * pad - KH) // stride + 1
    Wo = (W + 2 * pad - KW) // stride + 1
    a = torch.empty(B * Ho * Wo, ldk, dtype=BF16, device=x.device)
    with _span("stem_im2col", 0.0, x, a):
        _call("im2col_nchw", _p(x), _p(a), B, C, H, W, KH, KW, stride, pad, ldk)
    return a, Ho, Wo


# --------------------------------------------------------------------------------------------------------- conv / linear
def _conv2d_grouped_fwd(x, w_packed, ksize, stride, want_stats, act, groups, bn_scale=None, bn_shift=None):
    B, H, W, C = x.shape
    Ho, Wo = out_hw(H, ksize, stride), out_hw(W, ksize, stride)
    stats = None
    if want_stats:
        T = _query("conv2d_grouped_fwd_stats_rows", B, H, W, C, groups, ksize, stride)
        stats = torch.empty(T, 2, C, dtype=F32, device=x.device)
    y = torch.empty(B, Ho, Wo, C, dtype=BF16, device=x.device)
    with _span("conv_gemm_grouped_fwd", 2.0 * B * Ho * Wo * C * (C // groups) * ksize * ksize, x, w_packed, y):
        _call("conv2d_grouped_fwd", _p(x), _p(w_packed), _p(y), B, H, W, C, groups, ksize, stride, _p(stats), act,
              _p(bn_scale), _p(bn_shift))
    return y, stats


def conv2d_fwd(x, w_packed, ksize=1, stride=1, want_stats=False, bias=None, act=0, residual=None, out_f32=False, groups=1):
    """y = conv(x) (+bias)(act)(+residual). Returns (y, stats) with stats = [T,2,Cout] partial sums or None.
    groups > 1: grouped 3x3 convolution (w_packed = pack_weight(w, mode=3)); bias, residual and fp32 output are not offered."""
    _chk_act(x, "x")
    if groups != 1:
        if bias is not None or residual is not None or out_f32:
            raise ValueError("conv2d_fwd: a grouped convolution takes no bias, residual or fp32 output")
        return _conv2d_grouped_fwd(x, w_packed, ksize, stride, want_stats, act, groups)
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    Ho, Wo = out_hw(H, ksize, stride), out_hw(W, ksize, stride)
    stats = None
    if want_stats:
        T = _query("conv2d_fwd_stats_rows", B, H, W, Cout, ksize, stride)
        stats = torch.empty(T, 2, Cout, dtype=F32, device=x.device)
    y = torch.empty(B, Ho, Wo, Cout, dtype=F32 if out_f32 else BF16, device=x.device)
    with _span("conv_gemm_fwd", 2.0 * B * Ho * Wo * Cout * Cin * ksize * ksize, x, w_packed, y, residual):
        if out_f32:
            _call("conv2d_fwd", _p(x), _p(w_packed), None, B, H, W, Cin, Cout, ksize, stride, _p(stats), _p(bias), act,
                  _p(residual), _p(y), Cout, None, None)
        else:
            _call("conv2d_fwd", _p(x), _p(w_packed), _p(y), B, H, W, Cin, Cout, ksize, stride, _p(stats), _p(bias), act,
                  _p(residual), None, 0, None, None)
    return y, stats


def conv2d_bn_act(x, w_packed, co, ksize=1, stride=1, relu=True, residual=None, groups=1):
    """Eval-mode conv -> BatchNorm(fixed statistics) (-> + residual) (-> ReLU) as ONE implicit-GEMM launch: the BN scale / shift
    live in the epilogue, no BatchNorm pass at all.  groups > 1: grouped 3x3 convolution (pack_weight mode 3), no residual."""
    _chk_act(x, "x")
    if groups != 1:
        if residual is not None:
            raise ValueError("conv2d_bn_act: a grouped convolution takes no residual")
        return _conv2d_grouped_fwd(x, w_packed, ksize, stride, False, 1 if relu else 0, groups, co.scale, co.shift)[0]
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    Ho, Wo = out_hw(H, ksize, stride), out_hw(W, ksize, stride)
    y = torch.empty(B, Ho, Wo, Cout, dtype=BF16, device=x.device)
    with _span("conv_gemm_fwd", 2.0 * B * Ho * Wo * Cout * Cin * ksize * ksize, x, w_packed, y, residual):
        _call("conv2d_fwd", _p(x), _p(w_packed), _p(y), B, H, W, Cin, Cout, ksize, stride, None, None, 1 if relu else 0,
              _p(residual), None, 0, _p(co.scale), _p(co.shift))
    return y


def _bn_mask_arg(bn_mask, B, H, W, C, ksize, groups=1):
    """(BnMask, stats) for a dgrad / dual GEMM that masks its output with relu'(bn(x_raw)) and writes the BN-backward partial
    sums into stats; (None, None) without bn_mask."""
    if bn_mask is None:
        return None, None
    x_raw, co = bn_mask
    assert x_raw.dtype == BF16 and x_raw.is_contiguous() and x_raw.shape[-1] == C and C % 64 == 0
    if groups != 1:   # (the grouped kernel runs 64-channel tiles: its own row count)
        rows = _query("conv2d_grouped_fwd_stats_rows", B, H, W, C, groups, ksize, 1)
    else:
        rows = _query("conv2d_fwd_stats_rows", B, H, W, C, ksize, 1)
    stats = torch.empty(rows, 2, C, dtype=F32, device=x_raw.device)
    return _lib.BnMask(_p(x_raw), _p(co.scale), _p(co.shift), _p(stats)), stats


def conv2d_dgrad(dy, wd_packed, in_hw, ksize=1, stride=1, residual=None, out=None, bn_mask=None, groups=1):
    """dx[B,H,W,Cin] from dy[B,Ho,Wo,Cout]; wd_packed = pack_weight(w, mode=1). `out` lets 1x1/s2 accumulate in place.
    bn_mask = (x_raw, BnCoeffs) (stride 1): dx is the gradient of relu(bn(x_raw)); returns (dz, partial sums) for
    bn_backward_from_sums instead of dx.  groups > 1: grouped 3x3 convolution (wd_packed = pack_weight(w, mode=4)), no
    residual / out."""
    _chk_act(dy, "dy")
    B, Ho, Wo, Cout = dy.shape
    H, W = in_hw
    Cin = wd_packed.shape[0]
    if groups != 1:
        if residual is not None or out is not None:
            raise ValueError("conv2d_dgrad: a grouped convolution takes no residual or out")
        dx = torch.empty(B, H, W, Cin, dtype=BF16, device=dy.device)
        assert bn_mask is None or stride == 1, "bn_mask needs a stride-1 convolution"
        mask, stats = _bn_mask_arg(bn_mask, B, H, W, Cin, ksize, groups)
        with _span("conv_gemm_grouped_dgrad", 2.0 * B * Ho * Wo * Cout * (Cin // groups) * ksize * ksize,
                   dy, wd_packed, dx, bn_mask[0] if bn_mask else None):
            _call("conv2d_grouped_dgrad", _p(dy), _p(wd_packed), _p(dx), B, H, W, Cin, groups, ksize, stride, mask)
        return dx if bn_mask is None else (dx, stats)
    if out is not None:
        dx = out
    elif ksize == 1 and stride == 2:
        # a 1x1 / stride-2 convolution only reads the even input pixels: the kernel writes that phase alone, the gradient of
        # every other pixel is zero
        dx = torch.zeros(B, H, W, Cin, dtype=BF16, device=dy.device)
    else:
        dx = torch.empty(B, H, W, Cin, dtype=BF16, device=dy.device)
    assert bn_mask is None or stride == 1, "bn_mask needs a stride-1 convolution"
    mask, stats = _bn_mask_arg(bn_mask, B, H, W, Cin, ksize)
    with _span("conv_gemm_dgrad", 2.0 * B * Ho * Wo * Cout * Cin * ksize * ksize,
               dy, wd_packed, dx, residual, bn_mask[0] if bn_mask else None):
        _call("conv2d_dgrad", _p(dy), _p(wd_packed), _p(dx), B, H, W, Cin, Cout, ksize, stride, _p(residual), mask)
    return dx if bn_mask is None else (dx, stats)


_ws_cache = {}


def _workspace(nbytes, device):
    """Scratch of at least ``nbytes`` for the current stream.  Inside a CUDA-graph capture it is a fresh allocation from the
    graph's private pool: a cached buffer could be replaced (freed) by a larger request later in the same capture or in
    another graph captured on the same stream, while the graph that recorded its address is still replayed."""
    if torch.cuda.is_current_stream_capturing():
        return torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
    key = (device, torch.cuda.current_stream().cuda_stream)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = ws
    return ws


def conv2d_wgrad(dy, x, ksize=1, stride=1, out=None, accumulate=False, bias_out=None, groups=1):
    """dw fp32 OIHW [Cout, Cin, k, k] = sum over pixels of dy (x) x.
    bias_out (fp32 [Cout]): also write the bias gradient (column sums of dy), summed from the dy tiles the kernel already
    holds in shared memory - no extra pass over dy.  groups > 1: grouped 3x3 convolution, dw [C, C/groups, k, k]."""
    _chk_act(dy, "dy")
    _chk_act(x, "x")
    B, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    if groups != 1:
        if bias_out is not None:
            raise ValueError("conv2d_wgrad: a grouped convolution takes no bias gradient")
        nbytes = _query("conv2d_grouped_wgrad_workspace_bytes", B, H, W, Cin, groups, ksize, stride)
        ws = _workspace(nbytes, x.device)
        if out is None:
            out = torch.empty(Cout, Cin // groups, ksize, ksize, dtype=F32, device=x.device)
            accumulate = False
        with _span("wgrad_gemm_grouped", 2.0 * dy.numel() * (Cin // groups) * ksize * ksize, dy, x, out):
            _call("conv2d_grouped_wgrad", _p(dy), _p(x), _p(out), _p(ws), ws.numel(), B, H, W, Cin, groups, ksize, stride,
                  1 if accumulate else 0)
        return out
    nbytes = _query("conv2d_wgrad_workspace_bytes", B, H, W, Cin, Cout, ksize, stride)
    ws = _workspace(nbytes, x.device)
    if out is None:
        out = torch.empty(Cout, Cin, ksize, ksize, dtype=F32, device=x.device)
        accumulate = False
    bias_partial = None
    if bias_out is not None:   # finished by the split-reduction kernel of the same call
        splits = _query("conv2d_wgrad_splits", B, H, W, Cin, Cout, ksize, stride)
        bias_partial = torch.empty(splits, 2, Cout, dtype=F32, device=x.device)
    with _span("wgrad_gemm", 2.0 * dy.numel() * Cin * ksize * ksize, dy, x, out):
        _call("conv2d_wgrad", _p(dy), _p(x), _p(out), _p(ws), ws.numel(), B, H, W, Cin, Cout, ksize, stride,
              1 if accumulate else 0, _p(bias_partial), _p(bias_out))
    return out


# --------------------------------------------------------------------------------------------------------- batch norm
_scratch_cache = {}


def _reduce_scratch(device):
    """Persistent zero-initialised scratch for the two-level column reductions (ticket counters + slice sums), per stream."""
    key = (device, torch.cuda.current_stream().cuda_stream)
    sc = _scratch_cache.get(key)
    if sc is None:
        sc = torch.zeros(1024 + 64 * 2 * 8192 * 8, dtype=torch.uint8, device=device)
        _scratch_cache[key] = sc
    return sc


class BnCoeffs:
    """Per-channel vectors of one BatchNorm application (all fp32 [C])."""
    __slots__ = ("mean", "invstd", "scale", "shift")

    def __init__(self, C, device):
        buf = torch.empty(4, C, dtype=F32, device=device)
        self.mean, self.invstd, self.scale, self.shift = buf[0], buf[1], buf[2], buf[3]


def _sync_sums(partial, sync, average=False):
    """SyncBatchNorm (torch.nn.SyncBatchNorm of the DDP recipe, others/train_with_DDP/train.py:190): the rank's partial rows
    [T, 2, C] collapse to one row that is summed over the ranks of ``sync = (process_group, world_size)`` - one 2*C-float
    all-reduce per BatchNorm pass.  ``average`` divides by the world size: the backward pass then yields m1 / m2 of the GLOBAL
    batch from the local row count, and dgamma / dbeta equal to (global sum) / world on every rank, which the gradient
    all-reduce (SUM, scaled by 1 / world) turns into exactly the reference's averaged gradient."""
    import torch.distributed as dist

    group, world = sync
    row = partial.sum(0, keepdim=True)
    dist.all_reduce(row, op=dist.ReduceOp.SUM, group=group)
    if average:
        row.mul_(1.0 / world)
    return row


def bn_finalize(stats, count, gamma, beta, eps, momentum, running_mean, running_var, num_batches_tracked, sync=None):
    if sync is not None:
        stats = _sync_sums(stats, sync)
        count = count * sync[1]
    T, _, C = stats.shape
    co = BnCoeffs(C, stats.device)
    sc = _reduce_scratch(stats.device)
    _call("bn_finalize", _p(stats), T, C, float(count), _p(gamma), _p(beta), eps, momentum, _p(running_mean),
          _p(running_var), _p(num_batches_tracked), _p(co.mean), _p(co.invstd), _p(co.scale),
          _p(co.shift), _p(sc), sc.numel())
    return co


def bn_eval_coeffs(gamma, beta, running_mean, running_var, eps):
    C = gamma.numel()
    co = BnCoeffs(C, gamma.device)
    co.mean.copy_(running_mean)
    _call("bn_eval_coeffs", C, _p(gamma), _p(beta), _p(running_mean), _p(running_var), eps, _p(co.scale),
          _p(co.shift))
    return co


def bn_apply(x, co, relu=True, residual=None):
    C = x.shape[-1]
    rows = x.numel() // C
    y = torch.empty_like(x)
    with _span("bn_apply", 0.0, x, y, residual):
        _call("bn_apply", _p(x), _p(residual), _p(y), _p(co.scale), _p(co.shift), rows, C, 1 if relu else 0)
    return y


def bn_backward(g, x, co, relu=True, y_out=None, want_dz=False, dgamma=None, dbeta=None, accumulate=False, sync=None):
    """Train-mode BN (+ReLU) backward. g: grad wrt the post-activation output; x: raw conv output.
    Returns (dx, dgamma, dbeta, dz) with dz only when want_dz (masked upstream gradient, bf16)."""
    C = x.shape[-1]
    rows = x.numel() // C
    nblk = _query("bn_bwd_blocks", rows, C)
    partial = torch.empty(nblk, 2, C, dtype=F32, device=x.device)
    dz = torch.empty_like(x) if want_dz else None
    with _span("bn_bwd_reduce", 0.0, g, x, y_out, dz):
        _call("bn_bwd_reduce", _p(g), _p(x), _p(y_out), _p(dz), _p(co.scale), _p(co.shift), 1 if relu else 0, rows, C,
              _p(partial))
    if sync is not None:
        partial = _sync_sums(partial, sync, average=True)
    dgamma, dbeta, m = bn_bwd_finalize(partial, rows, co, dgamma, dbeta, accumulate)
    dx = torch.empty_like(x)
    src = dz if want_dz else g
    with _span("bn_bwd_apply", 0.0, src, x, dx, None if want_dz else y_out):
        _call("bn_bwd_apply", _p(src), _p(x), _p(y_out), 1 if want_dz else 0, _p(dx), _p(co.scale), _p(co.shift),
              _p(co.mean), _p(co.invstd), _p(m[0]), _p(m[1]), 1 if relu else 0, rows, C)
    return dx, dgamma, dbeta, dz


def bn_bwd_finalize(partial, count, co, dgamma=None, dbeta=None, accumulate=False):
    """dgamma, dbeta and m = {m1, m2} fp32 [2, C] of a train-mode BatchNorm from partial [T, 2, C] = {sum dz, sum dz * x}
    (x the raw BatchNorm input, co its BnCoeffs).  ``accumulate`` adds onto the given dgamma / dbeta."""
    T, _, C = partial.shape
    dev = partial.device
    acc = 1 if (accumulate and dgamma is not None) else 0
    if dgamma is None:
        dgamma = torch.empty(C, dtype=F32, device=dev)
    if dbeta is None:
        dbeta = torch.empty(C, dtype=F32, device=dev)
    m = torch.empty(2, C, dtype=F32, device=dev)
    sc = _reduce_scratch(dev)
    _call("bn_bwd_finalize", _p(partial), T, C, float(count), _p(dgamma), _p(dbeta), acc, _p(m[0]), _p(m[1]),
          _p(co.mean), _p(co.invstd), _p(sc), sc.numel())
    return dgamma, dbeta, m


def bn_backward_from_sums(dz, partial, x, co, dgamma=None, dbeta=None, sync=None):
    """Train-mode BatchNorm backward from a gradient dz that is already masked, bf16 shaped like x, and its partial sums
    [T, 2, C] = {sum dz, sum dz * x} (a dgrad / gemm_dual epilogue with bn_mask=, or a reduce pass): finalize, then
    dx = scale * (dz - m1 - xhat * m2) at any channel count that is a multiple of 8 up to 8192.  Returns (dx, dgamma, dbeta)."""
    _chk_act(dz, "dz")
    _chk_act(x, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    if sync is not None:
        partial = _sync_sums(partial, sync, average=True)
    dgamma, dbeta, m = bn_bwd_finalize(partial, rows, co, dgamma, dbeta)
    dx = torch.empty_like(x)
    with _span("bn_bwd_apply", 0.0, dz, x, dx):
        _call("bn_bwd_apply", _p(dz), _p(x), None, 1, _p(dx), _p(co.scale), _p(co.shift), _p(co.mean), _p(co.invstd),
              _p(m[0]), _p(m[1]), 1, rows, C)
    return dx, dgamma, dbeta


# ------------------------------------------------------------------------------ squeeze-and-excitation tail (csrc/se.cuh)
def _f32_param(w):
    w = w.detach()
    return w if (w.dtype == F32 and w.is_contiguous()) else w.float().contiguous()


def se_squeeze(c, co):
    """c: raw conv output bf16 [B,H,W,C]; co: BnCoeffs of the BatchNorm after it.  Returns (csum, pool), fp32 [B, C]:
    per-image channel sums of c and the mean of u = c * scale + shift (SELayer.avg_pool of the BatchNorm output)."""
    _chk_act(c, "c")
    B, H, W, C = c.shape
    out = torch.empty(2, B, C, dtype=F32, device=c.device)
    with _span("se_squeeze", float(c.numel()), c, out):
        _call("se_squeeze", _p(c), _p(co.scale), _p(co.shift), _p(out[0]), _p(out[1]), B, H * W, C)
    return out[0], out[1]


def se_excite(pool, w1, w2):
    """SELayer.fc on fp32 [B, C]: h = relu(pool w1^T) [B, Cr], gate = sigmoid(h w2^T) [B, C] (w1 [Cr, C], w2 [C, Cr])."""
    w1, w2 = _f32_param(w1), _f32_param(w2)
    B, C = pool.shape
    Cr = w1.shape[0]
    if tuple(w1.shape) != (Cr, C) or tuple(w2.shape) != (C, Cr):
        raise ValueError(f"se_excite: weights {tuple(w1.shape)} / {tuple(w2.shape)} do not match C={C}")
    h = torch.empty(B, Cr, dtype=F32, device=pool.device)
    gate = torch.empty(B, C, dtype=F32, device=pool.device)
    with _span("se_excite", 4.0 * B * C * Cr, pool, w1, w2, h, gate):
        _call("se_excite", _p(pool), _p(w1), _p(w2), _p(h), _p(gate), B, C, Cr)
    return h, gate


def se_apply(c, co, gate, identity):
    """y = relu((c * scale + shift) * gate[b] + identity), bf16 [B,H,W,C]: bn_apply with a per-(image, channel) multiplier."""
    _chk_act(c, "c")
    _chk_act(identity, "identity")
    B, H, W, C = c.shape
    y = torch.empty_like(c)
    with _span("se_apply", 0.0, c, identity, y):
        _call("se_apply", _p(c), _p(identity), _p(y), _p(co.scale), _p(co.shift), _p(gate), B, H * W, C)
    return y


def se_backward(g, y, c, co, csum, pool, h, gate, w1, w2, dw1=None, dw2=None, dgamma=None, dbeta=None):
    """Backward of y = relu(bn(c) * gate + identity) with the SE gate (train-mode BatchNorm), for g = dL/dy.
    Returns (dc, dz, dw1, dw2, dgamma, dbeta): dc = dL/dc, dz = dL/d(identity) (bf16); the four parameter gradients are
    written into the given buffers when passed (not accumulated)."""
    _chk_act(g, "g")
    w1, w2 = _f32_param(w1), _f32_param(w2)
    B, H, W, C = c.shape
    HW, Cr = H * W, w1.shape[0]
    dev = c.device
    dz = torch.empty_like(c)
    sums = torch.empty(2, B, C, dtype=F32, device=dev)
    with _span("se_bwd_reduce", 0.0, g, y, c, dz):
        _call("se_bwd_reduce", _p(g), _p(y), _p(c), _p(dz), _p(sums[0]), _p(sums[1]), B, HW, C)
    if dw1 is None:
        dw1 = torch.empty(Cr, C, dtype=F32, device=dev)
    if dw2 is None:
        dw2 = torch.empty(C, Cr, dtype=F32, device=dev)
    if dgamma is None:
        dgamma = torch.empty(C, dtype=F32, device=dev)
    if dbeta is None:
        dbeta = torch.empty(C, dtype=F32, device=dev)
    dh = torch.empty(B, Cr, dtype=F32, device=dev)
    dp = torch.empty(B, C, dtype=F32, device=dev)
    m = torch.empty(2, C, dtype=F32, device=dev)
    with _span("se_bwd_coeffs", 8.0 * B * C * Cr):
        _call("se_bwd_coeffs", _p(sums[0]), _p(sums[1]), _p(csum), _p(pool), _p(h), _p(gate), _p(w1), _p(w2), _p(co.scale),
              _p(co.shift), _p(co.mean), _p(co.invstd), B, HW, C, Cr, _p(dh), _p(dp), _p(dw1), _p(dw2),
              _p(dgamma), _p(dbeta), _p(m[0]), _p(m[1]))
    dc = torch.empty_like(c)
    with _span("se_bwd_apply", 0.0, dz, c, dc):
        _call("se_bwd_apply", _p(dz), _p(c), _p(dc), _p(gate), _p(dp), _p(co.scale), _p(co.mean), _p(co.invstd), _p(m[0]),
              _p(m[1]), B, HW, C)
    return dc, dz, dw1, dw2, dgamma, dbeta


# ------------------------------------------------------------------------------ RepVGG block passes (csrc/repvgg.cuh)
def _pitched(t, C, name):
    """(pointer, row pitch in elements, rows) of a bf16 CUDA tensor whose last dimension holds C channels and whose rows sit
    at one constant pitch (a contiguous tensor, or a channel slice [..., a:a+C] of one)."""
    if t.dtype != BF16 or not t.is_cuda or t.shape[-1] != C or t.stride(-1) != 1:
        raise ValueError(f"{name}: expected a CUDA bf16 tensor [..., {C}] with unit channel stride, got {t.dtype} "
                         f"{tuple(t.shape)} strides {t.stride()}")
    ld = t.stride(-2) if t.dim() >= 2 else C
    expect = ld
    for d in range(t.dim() - 2, -1, -1):
        if t.shape[d] != 1 and t.stride(d) != expect:
            raise ValueError(f"{name}: rows of {tuple(t.shape)} strides {t.stride()} are not evenly pitched")
        expect *= t.shape[d]
    return t.data_ptr(), ld, t.numel() // C


def repvgg_partial_rows(rows, C):
    """T: the number of [2][C] partial rows repvgg_apply(want_stats=True) and repvgg_bwd_reduce write for (rows, C)."""
    return _query("repvgg_partial_rows", rows, C)


def repvgg_apply(c3, c1, co3, co1, x=None, co_id=None, want_stats=False):
    """y = relu(bn3(c3) + bn1(c1) [+ bn_id(x)]) with BnCoeffs co3 / co1 / co_id, bf16 contiguous, shaped like c3.  c3, c1, x
    may be channel slices of wider tensors (the stem's [c3 | c1]).  Returns (y, stats) with stats fp32 [T, 2, C] = sums of
    the stored y and y^2 when want_stats, else None."""
    C = c3.shape[-1]
    p3, ld3, rows = _pitched(c3, C, "c3")
    p1, ld1, _ = _pitched(c1, C, "c1")
    px, ldx = (None, 0) if x is None else _pitched(x, C, "x")[:2]
    y = torch.empty(c3.shape, dtype=BF16, device=c3.device)
    stats = torch.empty(repvgg_partial_rows(rows, C), 2, C, dtype=F32, device=c3.device) if want_stats else None
    with _span("repvgg_apply", 0.0, c3, c1, x, y):
        _call("repvgg_apply", p3, ld3, p1, ld1, px, ldx, _p(co3.mean), _p(co1.mean), None if co_id is None else _p(co_id.mean),
              _p(y), rows, C, _p(stats))   # co.mean starts the BnCoeffs [4][C] buffer
    return y, stats


def repvgg_bwd_reduce(g, y, c3, c1, x=None):
    """dz = g * [y > 0]; returns partial fp32 [nb, T, 2, C] (nb = 2, or 3 with x): {sum dz, sum dz * input} per branch (dense,
    1x1, identity), each [T, 2, C] slab ready for bn_bwd_finalize."""
    _chk_act(g, "g")
    _chk_act(y, "y")
    C = y.shape[-1]
    p3, ld3, rows = _pitched(c3, C, "c3")
    p1, ld1, _ = _pitched(c1, C, "c1")
    px, ldx = (None, 0) if x is None else _pitched(x, C, "x")[:2]
    nb = 2 if x is None else 3
    partial = torch.empty(nb, repvgg_partial_rows(rows, C), 2, C, dtype=F32, device=y.device)
    with _span("repvgg_bwd_reduce", 0.0, g, y, c3, c1, x):
        _call("repvgg_bwd_reduce", _p(g), _p(y), p3, ld3, p1, ld1, px, ldx, rows, C, _p(partial))
    return partial


def repvgg_bwd_apply(g, y, c3, c1, co3, m3, co1, m1, x=None, co_id=None, m_id=None, out=None):
    """(dc3, dc1, dx): BatchNorm backward of every branch of y = relu(bn3(c3) + bn1(c1) [+ bn_id(x)]) for g = dL/dy, with m_*
    from bn_bwd_finalize.  dx (None without x) is the identity branch's data gradient.  ``out`` = (dc3, dc1, dx) buffers laid
    out like c3, c1, x (the stem writes [dc3 | dc1] into one tensor); by default each is allocated with its input's strides."""
    _chk_act(g, "g")
    _chk_act(y, "y")
    C = y.shape[-1]
    p3, ld3, rows = _pitched(c3, C, "c3")
    p1, ld1, _ = _pitched(c1, C, "c1")
    px, ldx = (None, 0) if x is None else _pitched(x, C, "x")[:2]
    if out is None:
        out = tuple(None if t is None else torch.empty_strided(t.shape, t.stride(), dtype=BF16, device=y.device)
                    for t in (c3, c1, x))
    for o, ld, name in ((out[0], ld3, "dc3"), (out[1], ld1, "dc1")) + (((out[2], ldx, "dx"),) if x is not None else ()):
        if _pitched(o, C, name)[1:] != (ld, rows):
            raise ValueError(f"repvgg_bwd_apply: {name} must have the row pitch of its input ({ld})")
    with _span("repvgg_bwd_apply", 0.0, g, y, c3, c1, x, out[0], out[1], out[2]):
        _call("repvgg_bwd_apply", _p(g), _p(y), p3, ld3, p1, ld1, px, ldx, _p(co3.mean), _p(m3), _p(co1.mean), _p(m1),
              None if co_id is None else _p(co_id.mean), _p(m_id), _p(out[0]), _p(out[1]), _p(out[2]),
              rows, C)
    return out


def _bn_fold_args(bn):
    if bn is None:
        return [None, None, None, None, 0.0]
    return [_p(bn.weight), _p(bn.bias), _p(bn.running_mean), _p(bn.running_var), float(bn.eps)]


def repvgg_fold(w3, w1, bn3, bn1, bn_id=None, ldk=None):
    """Eval-mode re-parameterisation of a RepVGG block from its fp32 parameters and running statistics: the bf16 forward
    operand [O][ldk] (k = tap * I + i, ldk defaults to 9 * I) of the equivalent 3x3 convolution and its fp32 bias [O]."""
    w3, w1 = _f32_param(w3), _f32_param(w1)
    O, I = w3.shape[0], w3.shape[1]
    if tuple(w3.shape) != (O, I, 3, 3) or w1.numel() != O * I:
        raise ValueError(f"repvgg_fold: weights {tuple(w3.shape)} / {tuple(w1.shape)} are not a 3x3 / 1x1 pair")
    ldk = 9 * I if ldk is None else ldk
    wp = torch.empty(O, ldk, dtype=BF16, device=w3.device)
    bias = torch.empty(O, dtype=F32, device=w3.device)
    _call("repvgg_fold", _p(w3), _p(w1), *_bn_fold_args(bn3), *_bn_fold_args(bn1), *_bn_fold_args(bn_id), O, I, ldk,
          _p(wp), _p(bias))
    return wp, bias


# ------------------------------------------------------------------------------ EfficientNet MBConv passes (csrc/mbconv.cuh)
def _dw_args(x, k, stride):
    _chk_act(x, "x")
    B, H, W, C = x.shape
    if k not in (3, 5) or stride not in (1, 2):
        raise ValueError(f"depthwise: k must be 3 or 5 and stride 1 or 2 (got k={k} stride={stride})")
    return B, H, W, C, (H - 1) // stride + 1, (W - 1) // stride + 1


def dw_fwd(x, w, k, stride, co=None, want_stats=False):
    """Depthwise k x k convolution (padding k // 2) of x bf16 [B,H,W,C] with the fp32 weight [C,1,k,k]; with BnCoeffs ``co``
    the input is silu(x * scale + shift) (the previous BatchNorm + SiLU applied on load).  Returns (d bf16 [B,Ho,Wo,C],
    stats fp32 [T,2,C] of the stored d, or None)."""
    B, H, W, C, Ho, Wo = _dw_args(x, k, stride)
    w = _f32_param(w)
    d = torch.empty(B, Ho, Wo, C, dtype=BF16, device=x.device)
    stats = None
    if want_stats:
        stats = torch.empty(_query("dw_partial_rows", B * Ho * Wo, C), 2, C, dtype=F32, device=x.device)
    with _span("dw_fwd", 2.0 * d.numel() * k * k, x, d):
        _call("dw_fwd", _p(x), _p(w), None if co is None else _p(co.scale), None if co is None else _p(co.shift), _p(d),
              _p(stats), B, H, W, C, k, stride)
    return d, stats


def dw_dgrad(dd, w, x, k, stride, co=None, residual=None):
    """Data gradient of dw_fwd for dd = dL/dd.  With BnCoeffs ``co`` (x the raw input normalised on load) returns
    (dz, partial): dz = g_in * silu'(x * scale + shift) bf16 and partial fp32 [T,2,C] = {sum dz, sum dz * x}; otherwise
    (g_in (+ residual), None)."""
    _chk_act(dd, "dd")
    B, H, W, C, Ho, Wo = _dw_args(x, k, stride)
    if tuple(dd.shape) != (B, Ho, Wo, C):
        raise ValueError(f"dw_dgrad: dd {tuple(dd.shape)} does not match the output of x {tuple(x.shape)}")
    w = _f32_param(w)
    dx = torch.empty_like(x)
    partial = None
    if co is not None:
        partial = torch.empty(_query("dw_partial_rows", B * H * W, C), 2, C, dtype=F32, device=x.device)
    with _span("dw_dgrad", 2.0 * dd.numel() * k * k, dd, x if co is not None else None, residual, dx):
        _call("dw_dgrad", _p(dd), _p(w), _p(x), None if co is None else _p(co.scale), None if co is None else _p(co.shift),
              _p(residual), _p(dx), _p(partial), B, H, W, C, k, stride)
    return dx, partial


def dw_wgrad(dd, x, k, stride, co=None, out=None):
    """Weight gradient fp32 [C, 1, k, k] of dw_fwd (``out`` receives it when given)."""
    _chk_act(dd, "dd")
    B, H, W, C, Ho, Wo = _dw_args(x, k, stride)
    nbytes = _query("dw_wgrad_workspace_bytes", B, H, W, C, k, stride)
    ws = _workspace(nbytes, x.device)
    if out is None:
        out = torch.empty(C, 1, k, k, dtype=F32, device=x.device)
    with _span("dw_wgrad", 2.0 * dd.numel() * k * k, dd, x):
        _call("dw_wgrad", _p(dd), _p(x), None if co is None else _p(co.scale), None if co is None else _p(co.shift),
              _p(out), _p(ws), nbytes, B, H, W, C, k, stride)
    return out


def silu_bn_squeeze(d, co, mask=None):
    """pool fp32 [B, C] = mean over pixels of silu(d * scale + shift); with ``mask`` fp32 [B, C] also returns the bf16
    [B, C] product pool * mask (the classifier input after dropout).  Returns (pool, masked or None)."""
    _chk_act(d, "d")
    B, H, W, C = d.shape
    pool = torch.empty(B, C, dtype=F32, device=d.device)
    out16 = torch.empty(B, C, dtype=BF16, device=d.device) if mask is not None else None
    if mask is not None:
        mask = mask.contiguous()
    with _span("silu_bn_squeeze", 0.0, d, pool):
        _call("silu_bn_squeeze", _p(d), _p(co.scale), _p(co.shift), _p(mask), _p(pool), _p(out16), B, H * W, C)
    return pool, out16


def excite_fwd(pool, w1, b1, w2, b2):
    """SELayer.fc with biases on fp32 [B, C]: hpre = pool w1^T + b1 [B, Cr], gate = sigmoid(silu(hpre) w2^T + b2) [B, C]."""
    B, C = pool.shape
    w1, w2, b1, b2 = _f32_param(w1), _f32_param(w2), _f32_param(b1), _f32_param(b2)
    Cr = w1.shape[0]
    if w1.numel() != Cr * C or w2.numel() != C * Cr or b1.numel() != Cr or b2.numel() != C:
        raise ValueError(f"excite_fwd: weights {tuple(w1.shape)} / {tuple(w2.shape)} do not match C={C}")
    hpre = torch.empty(B, Cr, dtype=F32, device=pool.device)
    gate = torch.empty(B, C, dtype=F32, device=pool.device)
    with _span("excite_fwd", 4.0 * B * C * Cr, pool, w1, w2, gate):
        _call("excite_fwd", _p(pool), _p(w1), _p(b1), _p(w2), _p(b2), _p(hpre), _p(gate), B, C, Cr)
    return hpre, gate


def excite_bwd(s, pool, hpre, gate, w1, w2, dw1=None, db1=None, dw2=None, db2=None):
    """Backward of excite_fwd from s = sum_p dL/da * silu(u) [B, C] (gate_reduce).  Returns (dpool [B, C], dw1 [Cr, C],
    db1 [Cr], dw2 [C, Cr], db2 [C]), written into the given buffers when passed."""
    B, C = pool.shape
    w1, w2 = _f32_param(w1), _f32_param(w2)
    Cr = w1.shape[0]
    dev = pool.device
    dw1 = torch.empty(Cr, C, dtype=F32, device=dev) if dw1 is None else dw1
    db1 = torch.empty(Cr, dtype=F32, device=dev) if db1 is None else db1
    dw2 = torch.empty(C, Cr, dtype=F32, device=dev) if dw2 is None else dw2
    db2 = torch.empty(C, dtype=F32, device=dev) if db2 is None else db2
    scratch = torch.empty(B, C + Cr, dtype=F32, device=dev)
    dpool = torch.empty(B, C, dtype=F32, device=dev)
    with _span("excite_bwd", 8.0 * B * C * Cr):
        _call("excite_bwd", _p(s), _p(pool), _p(hpre), _p(gate), _p(w1), _p(w2), _p(scratch), _p(scratch) + 4 * B * C,
              _p(dw1), _p(db1), _p(dw2), _p(db2), _p(dpool), B, C, Cr)
    return dpool, dw1, db1, dw2, db2


def gate_apply(d, co, gate):
    """a = silu(d * scale + shift) * gate[b] bf16 [B,H,W,C] (SELayer's x * y on the depthwise BatchNorm + SiLU output)."""
    _chk_act(d, "d")
    B, H, W, C = d.shape
    a = torch.empty_like(d)
    with _span("gate_apply", 0.0, d, a):
        _call("gate_apply", _p(d), _p(co.scale), _p(co.shift), _p(gate), _p(a), B, H * W, C)
    return a


def gate_reduce(da, d, co):
    """s fp32 [B, C] = sum over pixels of da * silu(d * scale + shift)."""
    _chk_act(da, "da")
    _chk_act(d, "d")
    B, H, W, C = d.shape
    s = torch.empty(B, C, dtype=F32, device=d.device)
    with _span("gate_reduce", 0.0, da, d):
        _call("gate_reduce", _p(da), _p(d), _p(co.scale), _p(co.shift), _p(s), B, H * W, C)
    return s


def silu_bn_bwd_reduce(d, co, dpool, da=None, gate=None):
    """dz = (da * gate + dpool / HW) * silu'(d * scale + shift) bf16 and partial fp32 [T,2,C] = {sum dz, sum dz * d}."""
    _chk_act(d, "d")
    B, H, W, C = d.shape
    dz = torch.empty_like(d)
    partial = torch.empty(repvgg_partial_rows(B * H * W, C), 2, C, dtype=F32, device=d.device)
    with _span("silu_bn_bwd_reduce", 0.0, da, d, dz):
        _call("silu_bn_bwd_reduce", _p(da), _p(gate), _p(dpool), _p(d), _p(co.scale), _p(co.shift), _p(dz), _p(partial),
              B, H * W, C)
    return dz, partial


def tail_apply(c, co, rs=None, residual=None):
    """y = (c * scale + shift) * rs[b] (+ residual) bf16: the project BatchNorm, drop-connect multiplier and shortcut."""
    _chk_act(c, "c")
    B, H, W, C = c.shape
    y = torch.empty_like(c)
    with _span("tail_apply", 0.0, c, residual, y):
        _call("tail_apply", _p(c), _p(co.scale), _p(co.shift), _p(rs), _p(residual), _p(y), B, H * W, C)
    return y


def tail_bwd_reduce(g, c, rs=None):
    """dz = g * rs[b] (g itself without rs) and partial fp32 [T,2,C] = {sum dz, sum dz * c}.  Returns (dz, partial)."""
    _chk_act(g, "g")
    _chk_act(c, "c")
    B, H, W, C = c.shape
    dz = torch.empty_like(g) if rs is not None else None
    partial = torch.empty(repvgg_partial_rows(B * H * W, C), 2, C, dtype=F32, device=c.device)
    with _span("tail_bwd_reduce", 0.0, g, c, dz):
        _call("tail_bwd_reduce", _p(g), _p(rs), _p(c), _p(dz), _p(partial), B, H * W, C)
    return (g if dz is None else dz), partial


# ------------------------------------------------------------------------------ BatchNorm folded through a 1x1 convolution
def gram_colsum(y2):
    """y2 bf16 [..., K] -> (G = y2^T y2 fp32 [K, K], s = column sums fp32 [K]): everything train-mode BatchNorm needs to know
    about the output of a 1x1 convolution of y2 (csrc/bn_algebra.cuh)."""
    K = y2.shape[-1]
    flat = y2.view(-1, 1, 1, K)
    # the column sums come from the tiles the Gram kernel already stages (its bias-gradient warps): no second pass over y2
    s = torch.empty(K, dtype=F32, device=y2.device)
    G = conv2d_wgrad(flat, flat, bias_out=s).view(K, K)
    return G, s


def bn_gram_stats(G, s, w_packed, count, gamma, beta, eps, momentum, running_mean, running_var, num_batches_tracked):
    """Batch statistics of conv1x1(y2, w) from (G, s); returns BnCoeffs and updates the running statistics."""
    N, K = w_packed.shape
    co = BnCoeffs(N, G.device)
    _call("bn_gram_stats", _p(G), _p(s), _p(w_packed), N, K, float(count), _p(gamma), _p(beta), eps, momentum,
          _p(running_mean), _p(running_var), _p(num_batches_tracked), _p(co.mean), _p(co.invstd),
          _p(co.scale), _p(co.shift))
    return co


def conv1x1_bn_act(x, w_packed, co, residual):
    """y = relu(conv1x1(x, w) * co.scale + co.shift + residual): conv + BatchNorm + identity + ReLU in one GEMM."""
    _chk_act(x, "x")
    _chk_act(residual, "residual")
    Cin = x.shape[-1]
    Cout = w_packed.shape[0]
    y = torch.empty(*x.shape[:-1], Cout, dtype=BF16, device=x.device)
    pixels = x.numel() // Cin
    with _span("conv_gemm_fwd", 2.0 * pixels * Cin * Cout, x, w_packed, residual, y):
        _call("conv1x1_bn_act_fwd", _p(x), _p(w_packed), _p(co.scale), _p(co.shift), _p(residual), _p(y), pixels, Cin, Cout, 1)
    return y


def conv1x1_bn(x, w_packed, co):
    """y = conv1x1(x, w) * co.scale + co.shift (downsample conv + BatchNorm in one GEMM; no residual, no ReLU)."""
    _chk_act(x, "x")
    Cin = x.shape[-1]
    Cout = w_packed.shape[0]
    y = torch.empty(*x.shape[:-1], Cout, dtype=BF16, device=x.device)
    pixels = x.numel() // Cin
    with _span("conv_gemm_fwd", 2.0 * pixels * Cin * Cout, x, w_packed, y):
        _call("conv1x1_bn_fwd", _p(x), _p(w_packed), _p(co.scale), _p(co.shift), _p(y), pixels, Cin, Cout)
    return y


def subsample2(x):
    """xs[b, i, j] = x[b, 2i, 2j]: the pixels a 1x1 / stride-2 convolution reads, as a compact NHWC tensor."""
    _chk_act(x, "x")
    B, H, W, C = x.shape
    xs = torch.empty(B, (H + 1) // 2, (W + 1) // 2, C, dtype=BF16, device=x.device)
    _call("subsample2", _p(x), _p(xs), B, H, W, C)
    return xs


def add_even_pixels_(gx, gs):
    """gx[b, 2i, 2j] += gs[b, i, j] in place."""
    B, H, W, C = gx.shape
    _call("add_even_pixels", _p(gx), _p(gs), B, H, W, C)
    return gx


def conv1x1_dgrad_masked(dy, wd_packed, residual, mask_src):
    """dz = (mask_src > 0) * (dy @ wd^T + residual); returns (dz bf16, stats fp32 [T,2,Cin] with plane 0 = partial sums of dz)."""
    _chk_act(dy, "dy")
    Cout = dy.shape[-1]
    Cin = wd_packed.shape[0]
    pixels = dy.numel() // Cout
    dz = torch.empty(*dy.shape[:-1], Cin, dtype=BF16, device=dy.device)
    T = _query("conv1x1_dgrad_masked_stats_rows", pixels, Cin, Cout)
    stats = torch.empty(T, 2, Cin, dtype=F32, device=dy.device)
    with _span("conv_gemm_dgrad", 2.0 * pixels * Cin * Cout, dy, wd_packed, residual, mask_src, dz):
        _call("conv1x1_dgrad_masked", _p(dy), _p(wd_packed), _p(dz), pixels, Cin, Cout, _p(residual), _p(mask_src), _p(stats))
    return dz, stats


def relu_mask_sum(g, y):
    """dz = (y > 0) * g with per-block partial column sums [T,2,C] (plane 0), for block outputs whose gradient does not come
    out of a masked dgrad epilogue (the BatchNorm-backward reduce pass with x = y; its second plane is unused)."""
    C = y.shape[-1]
    rows = y.numel() // C
    nblk = _query("bn_bwd_blocks", rows, C)
    partial = torch.empty(nblk, 2, C, dtype=F32, device=y.device)
    dz = torch.empty_like(y)
    with _span("bn_bwd_reduce", 0.0, g, y, dz):
        _call("bn_bwd_reduce", _p(g), _p(y), _p(y), _p(dz), None, None, 1, rows, C, _p(partial))
    return dz, partial


_ticket_cache = {}


def _algebra_tickets(device):
    """Persistent zero-initialised ticket counters of the M-tile reduction (per stream; the kernel leaves them zero)."""
    key = (device, torch.cuda.current_stream().cuda_stream)
    t = _ticket_cache.get(key)
    if t is None:
        t = torch.zeros(64, dtype=torch.int32, device=device)
        _ticket_cache[key] = t
    return t


def bn_conv1x1_bwd(dz_partial, D, G, s, w_packed, w_f32, count, gamma, co, dgamma=None, dbeta=None, dW=None):
    """BatchNorm + 1x1-conv backward algebra (csrc/bn_algebra.cuh). Returns (dgamma, dbeta, dW [N,K,1,1], wcat bf16 [K, N+K],
    bias fp32 [K]); wcat / bias are the operands of gemm_dual([dz | y2])."""
    N, K = w_packed.shape
    dev = D.device
    if dgamma is None:
        dgamma = torch.empty(N, dtype=F32, device=dev)
        dbeta = torch.empty(N, dtype=F32, device=dev)
    if dW is None:
        dW = torch.empty(N, K, 1, 1, dtype=F32, device=dev)
    wcat = torch.empty(K, N + K, dtype=BF16, device=dev)
    bias = torch.empty(K, dtype=F32, device=dev)
    nbytes = _query("bn_conv1x1_bwd_scratch_bytes", N, K)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    tickets = _algebra_tickets(dev)
    w32 = w_f32.detach()
    _call("bn_conv1x1_bwd", _p(dz_partial), dz_partial.shape[0], _p(D), _p(G), _p(s), _p(w_packed), _p(w32), N, K, float(count),
          _p(gamma), _p(co.mean), _p(co.invstd), _p(dgamma), _p(dbeta), _p(dW), 0, _p(wcat), _p(bias),
          _p(scratch), nbytes, _p(tickets))
    return dgamma, dbeta, dW, wcat, bias


def gemm_dual(a0, a1, wcat, bias, bn_mask=None):
    """out bf16 [..., N] = [a0 | a1] @ wcat^T + bias (a0 [..., K0], a1 [..., K1] bf16, wcat bf16 [N, K0 + K1]).
    bn_mask: as in conv2d_dgrad - returns (dz, partial sums)."""
    _chk_act(a0, "a0")
    _chk_act(a1, "a1")
    K0, K1 = a0.shape[-1], a1.shape[-1]
    N = wcat.shape[0]
    pixels = a0.numel() // K0
    out = torch.empty(*a0.shape[:-1], N, dtype=BF16, device=a0.device)
    mask, stats = _bn_mask_arg(bn_mask, 1, 1, pixels, N, 1)
    with _span("conv_gemm_dgrad", 2.0 * pixels * N * (K0 + K1), a0, a1, wcat, out, bn_mask[0] if bn_mask else None):
        _call("gemm_dual", _p(a0), K0, _p(a1), K1, _p(wcat), _p(bias), _p(out), pixels, N, mask)
    return out if bn_mask is None else (out, stats)


# --------------------------------------------------------------------------------------------------------- pooling
def bn_relu_maxpool_fwd(x, co):
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty(B, Ho, Wo, C, dtype=BF16, device=x.device)
    idx = torch.empty(B, Ho, Wo, C // 8, dtype=torch.int64, device=x.device)
    with _span("bn_relu_maxpool_fwd", 0.0, x, y, idx):
        _call("bn_relu_maxpool_fwd", _p(x), _p(y), _p(idx), _p(co.scale), _p(co.shift), B, H, W, C)
    return y, idx


def maxpool_bwd(g_out, idx, in_hw):
    B, Ho, Wo, C = g_out.shape
    H, W = in_hw
    g_in = torch.empty(B, H, W, C, dtype=BF16, device=g_out.device)
    with _span("maxpool_bwd", 0.0, g_out, idx, g_in):
        _call("maxpool_bwd", _p(g_out), _p(idx), _p(g_in), B, H, W, C)
    return g_in


def avgpool_fwd(x):
    B, H, W, C = x.shape
    y = torch.empty(B, C, dtype=BF16, device=x.device)
    _call("avgpool_fwd", _p(x), _p(y), B, H * W, C)
    return y


def avgpool_bwd(gy, hw):
    B, C = gy.shape
    H, W = hw
    gx = torch.empty(B, H, W, C, dtype=BF16, device=gy.device)
    _call("avgpool_bwd", _p(gy), _p(gx), B, H * W, C)
    return gx


# --------------------------------------------------------------------------------------------------------- loss / optimiser
def softmax_xent(logits, labels, want_grad=True, ld_d=None, label_smoothing=0.0, loss_scale=1.0):
    """Mean cross-entropy. Returns (loss scalar tensor, dlogits bf16 [B, ld_d] or None, correct int32 [B]).
    labels: int64 [B] class indices (optionally smoothed: LabelSmoothingCrossEntropy) or a floating [B, N] target
    distribution (SoftTargetCrossEntropy behind Mixup / CutMix).  loss_scale multiplies the GRADIENT only (1 / accumulation
    steps: swin_transformer/main.py:190)."""
    B, N = logits.shape
    ld_d = ld_d or ((N + 7) // 8) * 8
    rows = torch.empty(B, dtype=F32, device=logits.device)
    correct = torch.empty(B, dtype=torch.int32, device=logits.device)
    d = torch.empty(B, ld_d, dtype=BF16, device=logits.device) if want_grad else None
    gscale = float(loss_scale) / B
    if labels.is_floating_point():
        soft = labels if labels.dtype == F32 and labels.stride(1) == 1 else labels.float().contiguous()
        assert soft.shape == (B, N), f"soft targets must be [B, num_classes], got {tuple(soft.shape)}"
        _call("softmax_xent_soft", _p(logits), logits.stride(0), None, _p(soft), soft.stride(0), 0.0, B, N, gscale, _p(rows),
              _p(d), ld_d, _p(correct))
    elif label_smoothing > 0.0:
        _call("softmax_xent_soft", _p(logits), logits.stride(0), _p(labels), None, 0, float(label_smoothing), B, N, gscale,
              _p(rows), _p(d), ld_d, _p(correct))
    else:
        _call("softmax_xent", _p(logits), logits.stride(0), _p(labels), B, N, gscale, _p(rows), _p(d), ld_d,
              _p(correct))
    loss = torch.empty(1, dtype=F32, device=logits.device)
    _call("mean", _p(rows), B, _p(loss))
    return loss, d, correct


def colsum(m, cols=None, out=None, accumulate=False):
    rows, ld = m.shape
    cols = cols or ld
    if out is None:
        out = torch.empty(cols, dtype=F32, device=m.device)
        accumulate = False
    _call("colsum_bf16", _p(m), rows, ld, cols, _p(out), 1 if accumulate else 0)
    return out


def sgd_momentum_(p, g, buf, lr, momentum, weight_decay, gscale=1.0, first_step=False, lr_dev=None, clip=None):
    """lr_dev: optional 1-element fp32 CUDA tensor holding the learning rate (read by the kernel; graph friendly).
    clip: optional output of grad_clip_coef (the gradient is additionally scaled by clip[0])."""
    _call("sgd_momentum", _p(p), _p(g), _p(buf), p.numel(), float(lr), _p(lr_dev), momentum, weight_decay, gscale,
          1 if first_step else 0, _p(clip))


def stem_s2d(x):
    """fp32 NCHW [B,3,H,W] -> bf16 [B, H/2+3, W/2+3, 16] space-to-depth operand of the ResNet stem (see b200cls.h)."""
    B, C, H, W = x.shape
    if C != 3:
        raise ValueError("stem_s2d expects 3 input channels")
    z = torch.empty(B, H // 2 + 3, W // 2 + 3, 16, dtype=BF16, device=x.device)
    with _span("stem_s2d", 0.0, x, z):
        _call("stem_s2d", _p(x), _p(z), B, H, W)
    return z


IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)   # classification/resnet/train.py:51


def _f3(v):
    import ctypes

    return (ctypes.c_float * 3)(*[float(t) for t in v])


def stem_s2d_u8(x_u8, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """Decoded uint8 NHWC [B,H,W,3] -> the stem's space-to-depth operand, with ToTensor + Normalize fused in (GPU input pipeline)."""
    if x_u8.dtype != torch.uint8 or x_u8.dim() != 4 or x_u8.shape[-1] != 3 or not x_u8.is_cuda or not x_u8.is_contiguous():
        raise ValueError("stem_s2d_u8 expects a contiguous CUDA uint8 [B,H,W,3] batch")
    B, H, W, _ = x_u8.shape
    z = torch.empty(B, H // 2 + 3, W // 2 + 3, 16, dtype=BF16, device=x_u8.device)
    with _span("stem_s2d", 0.0, x_u8, z):
        _call("stem_s2d_u8", _p(x_u8), _p(z), B, H, W, _f3(mean), _f3(std))
    return z


def normalize_u8_nhwc(x_u8, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """Decoded uint8 NHWC [B,H,W,3] -> normalised fp32 NCHW [B,3,H,W] (ToTensor + Normalize on the GPU)."""
    B, H, W, _ = x_u8.shape
    y = torch.empty(B, 3, H, W, dtype=F32, device=x_u8.device)
    _call("normalize_u8_nhwc", _p(x_u8.contiguous()), _p(y), B, H, W, _f3(mean), _f3(std))
    return y


def stem_s2d_conv_fwd(z, w_packed, want_stats=False):
    """conv 7x7/2/pad 3 from the space-to-depth operand: returns (y bf16 [B,Ho,Wo,64], BN statistics partials or None)."""
    B, Hz, Wz, _ = z.shape
    Ho, Wo = Hz - 3, Wz - 3
    y = torch.empty(B, Ho, Wo, 64, dtype=BF16, device=z.device)
    stats = None
    if want_stats:
        stats = torch.empty(_query("conv2d_fwd_stats_rows", B, Ho, Wo, 64, 3, 1), 2, 64, dtype=F32, device=z.device)
    with _span("conv_gemm_fwd", 2.0 * B * Ho * Wo * 64 * 147, z, w_packed, y):
        _call("stem_s2d_conv_fwd", _p(z), _p(w_packed), _p(y), _p(stats), B, Ho, Wo)
    return y, stats


def stem_s2d_conv_wgrad(dy, z, out=None, accumulate=False):
    """Weight gradient [64,3,7,7] fp32 of the stem conv from dy bf16 [B,Ho,Wo,64] and the space-to-depth operand z."""
    B, Ho, Wo, _ = dy.shape
    ws = _workspace(_query("stem_s2d_conv_wgrad_workspace_bytes", B, Ho, Wo), dy.device)
    g = torch.empty(64, 64, 4, dtype=F32, device=dy.device)
    with _span("wgrad_gemm", 2.0 * dy.numel() * 147, dy, z):
        _call("stem_s2d_conv_wgrad", _p(dy), _p(z), _p(g), _p(ws), ws.numel() * ws.element_size(), B, Ho, Wo)
        if out is None:
            out = torch.empty(64, 3, 7, 7, dtype=F32, device=dy.device)
            accumulate = False
        _call("stem_s2d_wgrad_relayout", _p(g), _p(out), 1 if accumulate else 0)
    return out


def stem_wgrad_relayout(src, cout, cin, taps, out=None, accumulate=False):
    """[Cout][ldk] patch-matrix weight gradient (k = tap*Cin + c) -> OIHW [Cout, Cin, kh, kw] fp32."""
    ldk = src.shape[1]
    k = int(round(taps ** 0.5))
    if out is None:
        out = torch.empty(cout, cin, k, k, dtype=F32, device=src.device)
        accumulate = False
    _call("stem_wgrad_relayout", _p(src), _p(out), cout, cin, taps, ldk, 1 if accumulate else 0)
    return out


def launch_count():
    return _query("launch_count")


# --------------------------------------------------------------------------------------------------------- general GEMM
def _view(t, channels, pix_dims=None, pix_strides=None, offset=0):
    """b200_view_t of a tensor whose last dim is the channel dim (stride 1). Default: all leading dims flattened.
    `offset` (elements) moves the base, e.g. to skip the class-token row of a [B, T, D] tensor."""
    v = _lib.View()
    v.base = t.data_ptr() + offset * t.element_size()
    if pix_dims is None:
        rows = t.numel() // channels
        pix_dims, pix_strides = (rows, 1, 1), (channels, rows * channels, rows * channels)
    for i in range(3):
        v.dim[i] = int(pix_dims[i])
        v.stride[i] = int(pix_strides[i])
    return v


def gemm(a, w_packed, bias=None, act=0, out=None, out_f32=False, residual=None, aux_out=False, aux_in=None,
         a_view=None, out_view=None, residual_view=None, out_offset=0, want_stats=False, colscale=None, rowscale=None):
    """out[rows, N] = epilogue(a[rows, K] @ w_packed[N, K]^T). `*_view` = (pix_dims, pix_strides) for strided layouts.
    rowscale = (fp32 [n_samples] tensor, rows_per_sample): stochastic-depth multiplier of every sample's rows, applied
    before the residual add.  Returns (out, aux); with aux_out=True aux is the bf16 tensor the backward pass needs: GELU'(pre) for
    act=2 (the dgrad GEMM of the next layer multiplies by it: act=3, aux_in=aux), the pre-activation otherwise."""
    import ctypes

    N, K = w_packed.shape
    rows = a.numel() // K
    if out is None:
        out = torch.empty(*a.shape[:-1], N, dtype=F32 if out_f32 else BF16, device=a.device)
    out_f32 = out.dtype == F32
    av = _view(a, K, *(a_view or (None, None)))
    ov = _view(out, N, *(out_view or (None, None)), offset=out_offset)
    args = _lib.GemmArgs()
    args.w, args.N, args.K = w_packed.data_ptr(), N, K
    args.bias = _p(bias)
    args.colscale = _p(colscale)
    if rowscale is not None:
        args.rowscale, args.rows_per_sample = _p(rowscale[0]), int(rowscale[1])
    args.act = act
    args.out_f32 = 1 if out_f32 else 0
    keep = []
    if residual is not None:
        rv = _view(residual, N, *(residual_view or (None, None)))
        keep.append(rv)
        args.residual = ctypes.pointer(rv)
        args.residual_f32 = 1 if residual.dtype == F32 else 0
    aux = None
    if aux_out:
        aux = torch.empty(*a.shape[:-1], N, dtype=BF16, device=a.device)
        xv = _view(aux, N)
        keep.append(xv)
        args.aux_out = ctypes.pointer(xv)
    if aux_in is not None:
        iv = _view(aux_in, N)
        keep.append(iv)
        args.aux_in = ctypes.pointer(iv)
    stats = None
    if want_stats:
        # per-CTA column sums / sums of squares of the stored output (the BN-statistics epilogue): plane 0 summed over the
        # rows is e.g. the bias gradient of the layer whose output gradient this GEMM produces (see stats_colsum)
        if out_f32 or a_view is not None or out_view is not None:
            raise ValueError("gemm: want_stats needs a plain bf16 [rows, N] output")
        stats = torch.empty(_query("conv2d_fwd_stats_rows", rows, 1, 1, N, 1, 1), 2, N, dtype=F32, device=a.device)
        args.stats = _p(stats)
    with _span("conv_gemm_fwd", 2.0 * rows * N * K, a, w_packed, out, residual, aux, aux_in):
        _call("gemm_ex", ctypes.byref(av), ctypes.byref(ov), ctypes.byref(args))
    if want_stats:
        return out, aux, stats
    return out, aux


def stats_colsum(stats, out=None):
    """Column sums from epilogue statistics partials [T, 2, C] (plane 0): fp32 [C]."""
    T, _, C = stats.shape
    if out is None:
        out = torch.empty(C, dtype=F32, device=stats.device)
    sc = _reduce_scratch(stats.device)
    _call("bn_bwd_finalize", _p(stats), T, C, 1.0, None, _p(out), 0, None, None, None, None, _p(sc), sc.numel())
    return out


# --------------------------------------------------------------------------------------------------------- stochastic depth
def rowscale(x, scale):
    """y[b] = x[b] * scale[b] for a bf16 tensor whose first dim is the sample dim (scale fp32 [B])."""
    _chk_act(x, "x")
    B = scale.numel()
    per = x.numel() // B
    y = torch.empty_like(x)
    _call("rowscale_bf16", _p(x), _p(scale), _p(y), B, per)
    return y


def tanh_fwd(u):
    """fp32 u -> (t fp32, t bf16)."""
    t = torch.empty_like(u)
    t16 = torch.empty(u.shape, dtype=BF16, device=u.device)
    _call("tanh_fwd", _p(u), _p(t), _p(t16), u.numel())
    return t, t16


def tanh_bwd(dt16, t):
    du = torch.empty(t.shape, dtype=BF16, device=t.device)
    _call("tanh_bwd", _p(dt16), _p(t), _p(du), t.numel())
    return du


# --------------------------------------------------------------------------------------------------------- layer norm
# Widest rows the kernels take (b200_layernorm_fwd / _bwd, b200_patch_merge_ln_fwd / _bwd): the schedules reject a model
# with a wider LayerNorm before launching anything.
LAYERNORM_FWD_MAX_C = 3072
LAYERNORM_BWD_MAX_C = 1024
PATCH_MERGE_LN_MAX_C = 2048   # the merged width 4C


def layernorm_fwd(x, gamma, beta, eps, out_dtype=BF16):
    """x [..., C] fp32 or bf16 -> (y bf16 (or fp32), mean, rstd)."""
    C = x.shape[-1]
    rows = x.numel() // C
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    stat = torch.empty(2, rows, dtype=F32, device=x.device)
    with _span("layernorm_fwd", 0.0, x, y):
        _call("layernorm_fwd", _p(x), 1 if x.dtype == F32 else 0, _p(gamma), _p(beta), _p(y), 1 if out_dtype == F32 else 0,
              _p(stat[0]), _p(stat[1]), rows, C, eps)
    return y, stat[0], stat[1]


def layernorm_bwd(dy, x, mean, rstd, gamma, add=None, dx_dtype=BF16, dgamma=None, dbeta=None):
    """Returns (dx [+ add], dgamma, dbeta)."""
    C = x.shape[-1]
    rows = x.numel() // C
    nblk = _query("layernorm_bwd_blocks", rows, C)
    partial = torch.empty(nblk, 2, C, dtype=F32, device=x.device)
    dx = torch.empty(x.shape, dtype=dx_dtype, device=x.device)
    with _span("layernorm_bwd", 0.0, dy, x, dx, add):
        _call("layernorm_bwd", _p(dy), _p(x), 1 if x.dtype == F32 else 0, _p(mean), _p(rstd), _p(gamma), _p(add), _p(dx),
              1 if dx_dtype == F32 else 0, _p(partial), rows, C)
    if dgamma is None:
        dgamma = torch.empty(C, dtype=F32, device=x.device)
        dbeta = torch.empty(C, dtype=F32, device=x.device)
    sc = _reduce_scratch(x.device)
    _call("bn_bwd_finalize", _p(partial), nblk, C, 1.0, _p(dgamma), _p(dbeta), 0, None, None, None, None, _p(sc),
          sc.numel())
    return dx, dgamma, dbeta


# --------------------------------------------------------------------------------------------------------- ViT pieces
def patchify_nchw(x, ps):
    B, C, H, W = x.shape
    a = torch.empty(B, (H // ps) * (W // ps), C * ps * ps, dtype=BF16, device=x.device)
    with _span("patchify", 0.0, x, a):
        _call("patchify_nchw", _p(x), _p(a), B, C, H, W, ps)
    return a


def cls_row_(tokens, cls, pos):
    B, T, D = tokens.shape
    _call("cls_row", _p(cls), _p(pos), _p(tokens), B, T, D)


def batch_rowsum(g, stride_b, B, D, out=None, accumulate=False, offset=0):
    """out[d] (+)= sum_b g.flat[offset + b*stride_b + d]  (g fp32 or bf16)."""
    if out is None:
        out = torch.empty(D, dtype=F32, device=g.device)
        accumulate = False
    ptr = g.data_ptr() + offset * g.element_size()
    _call("batch_rowsum", ptr, 1 if g.dtype == F32 else 0, stride_b, B, D, _p(out), 1 if accumulate else 0)
    return out


def copy_rows(src, src_offset, src_pitch, dst, dst_offset, dst_pitch, rows, cols):
    """dst.flat[dst_offset + r*dst_pitch + c] = src.flat[src_offset + r*src_pitch + c] (same dtype; 16-byte granularity)."""
    es = src.element_size()
    _call("copy_rows", src.data_ptr() + src_offset * es, src_pitch * es, dst.data_ptr() + dst_offset * es,
          dst_pitch * es, rows, cols * es)


def colsum_tall(m, cols=None, out=None):
    """Column sums of a tall bf16 matrix [rows, ld] (bias gradients) using the two-level reduction."""
    rows, ld = m.shape
    cols = cols or ld
    S = _query("colsum_partial_slices", rows)
    partial = torch.empty(S, 2, cols, dtype=F32, device=m.device)
    _call("colsum_partial", _p(m), rows, ld, cols, _p(partial))
    if out is None:
        out = torch.empty(cols, dtype=F32, device=m.device)
    sc = _reduce_scratch(m.device)
    _call("bn_bwd_finalize", _p(partial), S, cols, 1.0, None, _p(out), 0, None, None, None, None, _p(sc), sc.numel())
    return out


def attention_fwd(qkv, H, scale):
    """qkv bf16 [B, T, 3*H*64] -> (out bf16 [B, T, H*64], lse fp32 [B, H, T])."""
    B, T, _ = qkv.shape
    out = torch.empty(B, T, H * 64, dtype=BF16, device=qkv.device)
    lse = torch.empty(B, H, T, dtype=F32, device=qkv.device)
    with _span("attention_fwd", 4.0 * B * H * T * T * 64, qkv, out):
        _call("attention_fwd", _p(qkv), _p(out), _p(lse), B, T, H, scale)
    return out, lse


def attention_bwd(qkv, out, dout, lse, H, scale):
    B, T, _ = qkv.shape
    dqkv = torch.empty_like(qkv)
    delta = torch.empty(B, H, T, dtype=F32, device=qkv.device)
    with _span("attention_bwd", 10.0 * B * H * T * T * 64, qkv, out, dout, dqkv):
        _call("attention_bwd", _p(qkv), _p(out), _p(dout), _p(lse), _p(delta), _p(dqkv), B, T, H, scale)
    return dqkv


# --------------------------------------------------------------------------------------------------------- ConvNeXt pieces
def dwconv7_pack(w):
    """[C,1,7,7] fp32 parameter -> tap-major [49, C] fp32 copy."""
    C = w.shape[0]
    wt = torch.empty(49, C, dtype=F32, device=w.device)
    _call("dwconv7_pack", _p(w.detach()), _p(wt), C)
    return wt


def dwconv7(x, wt, bias=None, add=None, out_dtype=BF16, flip=False):
    """7x7 depthwise conv (pad 3) on NHWC x; flip=True is the data-gradient (correlation with the flipped kernel)."""
    B, H, W, C = x.shape
    out = torch.empty(B, H, W, C, dtype=out_dtype, device=x.device)
    with _span("dwconv7", 2.0 * 49 * x.numel(), x, out, add):
        _call("dwconv7", _p(x), 1 if x.dtype == F32 else 0, _p(wt), _p(bias), _p(add), _p(out), 1 if out_dtype == F32 else 0,
              1 if flip else 0, B, H, W, C)
    return out


def dwconv7_wgrad(du, x, out=None, accumulate=False):
    """dw [C,1,7,7] = sum_pixels du * x_shifted (du bf16, x fp32, both NHWC)."""
    B, H, W, C = x.shape
    nbytes = _query("dwconv7_wgrad_workspace_bytes", B, H, W, C)
    ws = _workspace(nbytes, x.device)
    if out is None:
        out = torch.empty(C, 1, 7, 7, dtype=F32, device=x.device)
        accumulate = False
    with _span("dwconv7_wgrad", 2.0 * 49 * x.numel(), du, x):
        _call("dwconv7_wgrad", _p(du), _p(x), _p(out), _p(ws), ws.numel(), B, H, W, C, 1 if accumulate else 0)
    return out


def avgpool_any(x):
    """[B, H, W, C] (fp32 or bf16) -> fp32 [B, C] mean over H*W."""
    B, H, W, C = x.shape
    y = torch.empty(B, C, dtype=F32, device=x.device)
    _call("avgpool_any", _p(x), 1 if x.dtype == F32 else 0, _p(y), B, H * W, C)
    return y


def colsum_prod(a, b=None, out=None):
    """Column sums of a*b (bf16 [rows, C] each; b optional)."""
    rows, C = a.shape
    S = _query("colsum_partial_slices", rows)
    partial = torch.empty(S, 2, C, dtype=F32, device=a.device)
    _call("colsum_prod_partial", _p(a), _p(b), rows, C, C, _p(partial))
    if out is None:
        out = torch.empty(C, dtype=F32, device=a.device)
    sc = _reduce_scratch(a.device)
    _call("bn_bwd_finalize", _p(partial), S, C, 1.0, None, _p(out), 0, None, None, None, None, _p(sc), sc.numel())
    return out


def adamw_(p, g, m, v, wd, hyper, beta1=0.9, beta2=0.999, eps=1e-8, gscale=1.0, tick=True, clip=None):
    """hyper: fp32 CUDA tensor {lr, 1-beta1^t, 1-beta2^t, beta1^t, beta2^t} (init {lr, 0, 0, 1, 1}); tick advances t first.
    clip: optional output of grad_clip_coef (the gradient is additionally scaled by clip[0])."""
    if tick:
        _call("adamw_tick", _p(hyper), beta1, beta2)
    _call("adamw", _p(p), _p(g), _p(m), _p(v), _p(wd), p.numel(), _p(hyper), beta1, beta2, eps, gscale, _p(clip))


def grad_clip_coef(g, max_norm, gscale=1.0, out=None, scratch=None):
    """clip_grad_norm_ without touching the gradients: returns fp32 [2] = {min(1, max_norm / (gscale*||g|| + 1e-6)), norm}."""
    if out is None:
        out = torch.empty(2, dtype=F32, device=g.device)
    if scratch is None:
        scratch = torch.empty(_query("grad_clip_blocks"), dtype=F32, device=g.device)
    _call("grad_clip_coef", _p(g), g.numel(), float(gscale), float(max_norm), _p(scratch), _p(out))
    return out


def layerscale_grads(G, W2, b2, gsum, gamma, dW2=None, db2=None, dgamma=None):
    C, K = W2.shape
    dW2 = torch.empty(C, K, dtype=F32, device=G.device) if dW2 is None else dW2
    db2 = torch.empty(C, dtype=F32, device=G.device) if db2 is None else db2
    dgamma = torch.empty(C, dtype=F32, device=G.device) if dgamma is None else dgamma
    _call("layerscale_grads", _p(G), _p(W2), _p(b2), _p(gsum), _p(gamma), _p(dW2), _p(db2), _p(dgamma), C, K)
    return dW2, db2, dgamma


def conv2d_fwd_f32(x, w_packed, ksize, stride, bias=None):
    """Convolution with fp32 NHWC output (+bias): feeds the fp32 residual stream (ConvNeXt 2x2/s2 downsample)."""
    _chk_act(x, "x")
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    Ho, Wo = out_hw(H, ksize, stride), out_hw(W, ksize, stride)
    y = torch.empty(B, Ho, Wo, Cout, dtype=F32, device=x.device)
    with _span("conv_gemm_fwd", 2.0 * B * Ho * Wo * Cout * Cin * ksize * ksize, x, w_packed, y):
        _call("conv2d_fwd_f32", _p(x), _p(w_packed), _p(y), B, H, W, Cin, Cout, ksize, stride, _p(bias))
    return y


# --------------------------------------------------------------------------------------------------------- Swin pieces
def window_bias_gather(table, index, nH, mask=None):
    """relative_position_bias_table [(2*7-1)^2, nH] + relative_position_index [49,49] int64 (+ attn_mask [nW,49,49]) ->
    fp32 table [nH, nW or 1, 49 (query), 64 (key, 49 used)] read by the window-attention kernels."""
    nW = mask.shape[0] if mask is not None else 1
    tab = torch.empty(nH, nW, 49, 64, dtype=F32, device=table.device)
    _call("window_bias_gather", _p(table), _p(index), _p(mask), nW, _p(tab), nH)
    return tab


def window_bias_scatter(dbias, index, dtable):
    nH = dbias.shape[0]
    _call("window_bias_scatter", _p(dbias), _p(index), _p(dtable), nH)
    return dtable


def _wattn_masked(bias_tab, nW):
    """1 when the table carries one (bias + mask) slice per window; with a single window slice 0 is the right one anyway."""
    if bias_tab.shape[1] not in (1, nW):
        raise ValueError(f"window attention: bias table holds {bias_tab.shape[1]} window slices, the image has {nW} windows")
    return 1 if (bias_tab.shape[1] == nW and nW > 1) else 0


def window_attention_fwd(qkv, nH, bias_tab, shift, scale):
    """qkv bf16 [B,H,W,3*nH*32] (natural pixel order), bias_tab = window_bias_gather(...) ->
    (out bf16 [B,H,W,nH*32], lse fp32 [B,nW,nH,49])."""
    B, H, W, _ = qkv.shape
    C = nH * 32
    nW = (H // 7) * (W // 7)
    out = torch.empty(B, H, W, C, dtype=BF16, device=qkv.device)
    lse = torch.empty(B, nW, nH, 49, dtype=F32, device=qkv.device)
    with _span("window_attention_fwd", 4.0 * B * nW * nH * 49 * 49 * 32, qkv, out):
        _call("window_attention_fwd", _p(qkv), _p(out), _p(bias_tab), _wattn_masked(bias_tab, nW), _p(lse), B, H, W, nH, shift,
              scale)
    return out, lse


def window_attention_bwd(qkv, out, dout, bias_tab, lse, nH, shift, scale):
    """Returns (dqkv bf16 like qkv, dbias fp32 [nH,49,49])."""
    B, H, W, _ = qkv.shape
    nW = (H // 7) * (W // 7)
    dqkv = torch.empty_like(qkv)
    dbias = torch.zeros(nH, 49, 49, dtype=F32, device=qkv.device)
    with _span("window_attention_bwd", 10.0 * B * nW * nH * 49 * 49 * 32, qkv, out, dout, dqkv):
        _call("window_attention_bwd", _p(qkv), _p(out), _p(dout), _p(bias_tab), _wattn_masked(bias_tab, nW), _p(lse), _p(dqkv),
              _p(dbias), B, H, W, nH, shift, scale)
    return dqkv, dbias


def window_partition(x, shift, ws):
    """window_partition(torch.roll(x, (shift, shift), (1, 2))): [B,H,W,C] -> [B*nW, ws, ws, C] (any 2/4-byte dtype)."""
    B, H, W, C = x.shape
    out = torch.empty(B * (H // ws) * (W // ws), ws, ws, C, dtype=x.dtype, device=x.device)
    _call("window_partition", _p(x), _p(out), B, H, W, C, shift, ws, x.element_size())
    return out


def window_merge(xw, B, H, W, shift, ws):
    """torch.roll(window_reverse(xw), (shift, shift), (1, 2)): [B*nW, ws, ws, C] -> [B,H,W,C]."""
    C = xw.shape[-1]
    out = torch.empty(B, H, W, C, dtype=xw.dtype, device=xw.device)
    _call("window_merge", _p(xw), _p(out), B, H, W, C, shift, ws, xw.element_size())
    return out


def patch_merge_ln_fwd(x, gamma, beta, eps):
    """x fp32 [B,H,W,C] -> (y bf16 [B*H/2*W/2, 4C] = LN(concat 2x2), mean, rstd)."""
    B, H, W, C = x.shape
    rows = B * (H // 2) * (W // 2)
    y = torch.empty(rows, 4 * C, dtype=BF16, device=x.device)
    stat = torch.empty(2, rows, dtype=F32, device=x.device)
    with _span("patch_merge_ln_fwd", 0.0, x, y):
        _call("patch_merge_ln_fwd", _p(x), _p(gamma), _p(beta), _p(y), _p(stat[0]), _p(stat[1]), B, H, W, C, eps)
    return y, stat[0], stat[1]


def patch_merge_ln_bwd(dy, x, mean, rstd, gamma, dgamma=None, dbeta=None):
    """Returns (dx bf16 [B,H,W,C], dgamma, dbeta)."""
    B, H, W, C = x.shape
    rows = B * (H // 2) * (W // 2)
    nblk = _query("patch_merge_ln_bwd_blocks", rows)
    partial = torch.empty(nblk, 2, 4 * C, dtype=F32, device=x.device)
    dx = torch.empty(B, H, W, C, dtype=BF16, device=x.device)
    with _span("patch_merge_ln_bwd", 0.0, dy, x, dx):
        _call("patch_merge_ln_bwd", _p(dy), _p(x), _p(mean), _p(rstd), _p(gamma), _p(dx), _p(partial), B, H, W, C)
    if dgamma is None:
        dgamma = torch.empty(4 * C, dtype=F32, device=x.device)
        dbeta = torch.empty(4 * C, dtype=F32, device=x.device)
    sc = _reduce_scratch(x.device)
    _call("bn_bwd_finalize", _p(partial), nblk, 4 * C, 1.0, _p(dgamma), _p(dbeta), 0, None, None, None, None, _p(sc),
          sc.numel())
    return dx, dgamma, dbeta


# ------------------------------------------------------------------------------------------------- VGG passes (csrc/vgg.cuh)
def vgg_pool_fwd(x, co=None, want_idx=True):
    """MaxPool2d(2, 2) of x (plain: x = relu(conv + b)) or of relu(x * scale + shift) (co = BnCoeffs: x the raw conv output).
    Returns (y [B, H/2, W/2, C], idx uint8 of y's shape or None): idx holds the window tap of each maximum."""
    _chk_act(x, "x")
    B, H, W, C = x.shape
    y = torch.empty(B, H // 2, W // 2, C, dtype=BF16, device=x.device)
    idx = torch.empty(y.shape, dtype=torch.uint8, device=x.device) if want_idx else None
    with _span("vgg_pool_fwd", 0.0, x, y, idx):
        _call("vgg_pool_fwd", _p(x), _p(co.scale) if co else None, _p(co.shift) if co else None, _p(y), _p(idx), B, H, W, C)
    return y, idx


def vgg_pool_bwd(g, idx, in_hw, y=None, c=None, co=None):
    """Gradient [B, H, W, C] of vgg_pool_fwd's input from the pooled gradient g: plain (y = the pooled output) returns dx;
    BN (c = the raw conv output, co its BnCoeffs) returns (dz, partial [T, 2, C] = {sum dz, sum dz c})."""
    _chk_act(g, "g")
    B, _, _, C = g.shape
    H, W = in_hw
    dx = torch.empty(B, H, W, C, dtype=BF16, device=g.device)
    partial = None
    if c is not None:
        T = _query("vgg_pool_partial_rows", B, H, W, C)
        partial = torch.empty(T, 2, C, dtype=F32, device=g.device)
    with _span("vgg_pool_bwd", 0.0, g, idx, y, c, dx):
        _call("vgg_pool_bwd", _p(g), _p(idx), _p(y), _p(c), _p(co.scale) if co else None, _p(co.shift) if co else None,
              _p(dx), _p(partial), B, H, W, C)
    return dx if c is None else (dx, partial)


def vgg_avgpool7_fwd(x):
    """AdaptiveAvgPool2d((7, 7)) + torch.flatten of NHWC x: bf16 [B, C * 49] in NCHW flatten order (k = c * 49 + i * 7 + j)."""
    _chk_act(x, "x")
    B, H, W, C = x.shape
    y = torch.empty(B, C * 49, dtype=BF16, device=x.device)
    with _span("vgg_avgpool7_fwd", 0.0, x, y):
        _call("vgg_avgpool7_fwd", _p(x), _p(y), B, H, W, C)
    return y


def vgg_avgpool7_bwd(gy, in_shape):
    """Gradient [B, H, W, C] of vgg_avgpool7_fwd's input from gy [B, C * 49]."""
    _chk_act(gy, "gy")
    B, H, W, C = in_shape
    gx = torch.empty(B, H, W, C, dtype=BF16, device=gy.device)
    with _span("vgg_avgpool7_bwd", 0.0, gy, gx):
        _call("vgg_avgpool7_bwd", _p(gy), _p(gx), B, H, W, C)
    return gx


def vgg_dropout_fwd(x, mask):
    """x * mask (bf16 x, fp32 mask of x's shape: 0 or 1 / (1 - p))."""
    _chk_act(x, "x")
    mask = mask.contiguous()
    assert mask.dtype == F32 and mask.shape == x.shape
    y = torch.empty_like(x)
    _call("vgg_dropout_fwd", _p(x), _p(mask), _p(y), x.numel())
    return y


def vgg_dropout_bwd(g, h, p):
    """Gradient of pre in h = dropout_p(relu(pre)) from dL/dh and the stored h: h > 0 ? g / (1 - p) : 0."""
    _chk_act(g, "g")
    _chk_act(h, "h")
    dx = torch.empty_like(g)
    _call("vgg_dropout_bwd", _p(g), _p(h), 1.0 / (1.0 - p), _p(dx), g.numel())
    return dx


def adam_(p, g, m, v, hyper, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, gscale=1.0, tick=True, clip=None):
    """torch.optim.Adam step (L2 decay added to the gradient) over flat fp32 tensors; hyper as adamw_'s, tick advances t first.
    clip: optional output of grad_clip_coef (the gradient is additionally scaled by clip[0])."""
    if tick:
        _call("adamw_tick", _p(hyper), beta1, beta2)
    _call("adam", _p(p), _p(g), _p(m), _p(v), p.numel(), _p(hyper), beta1, beta2, eps, weight_decay, gscale, _p(clip))


# ------------------------------------------------------------------------------ ShuffleNet v1 passes (csrc/shufflenet.cuh)
def dw_relu_fwd(x, w, stride, co, want_stats=False):
    """3x3 depthwise convolution (padding 1) of relu(x * scale + shift) (BnCoeffs ``co``: the previous BatchNorm + ReLU
    applied on load), fp32 weight [C, 1, 3, 3].  Returns (d bf16 [B,Ho,Wo,C], stats fp32 [T,2,C] of the stored d, or None)."""
    B, H, W, C, Ho, Wo = _dw_args(x, 3, stride)
    w = _f32_param(w)
    d = torch.empty(B, Ho, Wo, C, dtype=BF16, device=x.device)
    stats = None
    if want_stats:
        stats = torch.empty(_query("dw_partial_rows", B * Ho * Wo, C), 2, C, dtype=F32, device=x.device)
    with _span("dw_relu_fwd", 18.0 * d.numel(), x, d):
        _call("dw_relu_fwd", _p(x), _p(w), _p(co.scale), _p(co.shift), _p(d), _p(stats), B, H, W, C, stride)
    return d, stats


def dw_relu_dgrad(dd, w, x, stride, co):
    """Data gradient of dw_relu_fwd for dd = dL/dd: (dz, partial) with dz = g_in * [x * scale + shift > 0] bf16 and
    partial fp32 [T,2,C] = {sum dz, sum dz * x}, the rows bn_bwd_finalize reads for the BatchNorm applied on load."""
    _chk_act(dd, "dd")
    B, H, W, C, Ho, Wo = _dw_args(x, 3, stride)
    if tuple(dd.shape) != (B, Ho, Wo, C):
        raise ValueError(f"dw_relu_dgrad: dd {tuple(dd.shape)} does not match the output of x {tuple(x.shape)}")
    w = _f32_param(w)
    dx = torch.empty_like(x)
    partial = torch.empty(_query("dw_partial_rows", B * H * W, C), 2, C, dtype=F32, device=x.device)
    with _span("dw_relu_dgrad", 18.0 * dd.numel(), dd, x, dx):
        _call("dw_relu_dgrad", _p(dd), _p(w), _p(x), _p(co.scale), _p(co.shift), _p(dx), _p(partial), B, H, W, C, stride)
    return dx, partial


def dw_relu_wgrad(dd, x, stride, co, out=None):
    """Weight gradient fp32 [C, 1, 3, 3] of dw_relu_fwd (``out`` receives it when given)."""
    _chk_act(dd, "dd")
    B, H, W, C, Ho, Wo = _dw_args(x, 3, stride)
    nbytes = _query("dw_wgrad_workspace_bytes", B, H, W, C, 3, stride)
    ws = _workspace(nbytes, x.device)
    if out is None:
        out = torch.empty(C, 1, 3, 3, dtype=F32, device=x.device)
    with _span("dw_relu_wgrad", 18.0 * dd.numel(), dd, x):
        _call("dw_relu_wgrad", _p(dd), _p(x), _p(co.scale), _p(co.shift), _p(out), _p(ws), nbytes, B, H, W, C, stride)
    return out


def shuffle_tail_s2_fwd(x, c3, co):
    """Stride-2 ShuffleNet block output bf16 [B,Ho,Wo,Cin+Cc] = cat(relu(avg_pool3x3/2/p1(x)), relu(c3 * scale + shift))."""
    _chk_act(x, "x")
    _chk_act(c3, "c3")
    B, H, W, Cin = x.shape
    Cc = c3.shape[-1]
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if tuple(c3.shape) != (B, Ho, Wo, Cc):
        raise ValueError(f"shuffle_tail_s2_fwd: c3 {tuple(c3.shape)} does not match the pooled x {(B, Ho, Wo)}")
    y = torch.empty(B, Ho, Wo, Cin + Cc, dtype=BF16, device=x.device)
    with _span("shuffle_tail_s2_fwd", 0.0, x, c3, y):
        _call("shuffle_tail_s2_fwd", _p(x), _p(c3), _p(co.scale), _p(co.shift), _p(y), B, H, W, Cin, Cc)
    return y


def shuffle_relu_bwd(g, c, y=None, co=None, in_hw=None):
    """ReLU-masked gradient of a ShuffleNet BatchNorm output c (bf16 [B,Ho,Wo,Cc]).  Returns (dz, partial, gx):
    dz = g * mask bf16 [B,Ho,Wo,Cc], partial fp32 [T,2,Cc] = {sum dz, sum dz * c}.
    - y given (block output, [B,Ho,Wo,Cin+Cc], g of the same shape): mask = y[..., Cin:] > 0.  With Cin > 0 (stride-2
      tail, ``in_hw`` = (H, W) of the block input) gx bf16 [B,H,W,Cin] is the avg-pool backward of g * [y > 0] over the
      first Cin channels; else gx is None.
    - co given (stem): mask = c * scale + shift > 0, g shaped like c."""
    _chk_act(g, "g")
    _chk_act(c, "c")
    B, Ho, Wo, Cc = c.shape
    Cin = 0 if y is None else y.shape[-1] - Cc
    if y is not None:
        _chk_act(y, "y")
        if tuple(g.shape) != tuple(y.shape) or tuple(y.shape[:3]) != (B, Ho, Wo):
            raise ValueError(f"shuffle_relu_bwd: g {tuple(g.shape)} / y {tuple(y.shape)} / c {tuple(c.shape)} disagree")
    elif tuple(g.shape) != tuple(c.shape):
        raise ValueError(f"shuffle_relu_bwd: g {tuple(g.shape)} must be shaped like c {tuple(c.shape)}")
    H, W = in_hw if Cin > 0 else (0, 0)
    dz = torch.empty_like(c)
    partial = torch.empty(repvgg_partial_rows(B * Ho * Wo, Cc), 2, Cc, dtype=F32, device=c.device)
    gx = torch.empty(B, H, W, Cin, dtype=BF16, device=c.device) if Cin > 0 else None
    with _span("shuffle_relu_bwd", 0.0, g, y, c, dz, gx):
        _call("shuffle_relu_bwd", _p(g), _p(y), _p(c), None if co is None else _p(co.scale),
              None if co is None else _p(co.shift), _p(dz), _p(partial), _p(gx), B, Ho, Wo, Cin, Cc, H, W)
    return dz, partial, gx


# ------------------------------------------------------------------------------ ShuffleNet v2 tails (csrc/shufflenet.cuh)
def _v2_pitch(b):
    return (2 * b + 7) // 8 * 8


def shufflev2_tail_fwd(u, c3, co, b, co_u=None, split=False):
    """channel_shuffle(cat(u, v), 2) of a ShuffleNet v2 block with v = relu(c3 * scale + shift) (BnCoeffs ``co``) and u the
    passthrough half, or relu(u * scale + shift) with BnCoeffs ``co_u`` (u then branch1's raw GEMM output).  u, c3 bf16
    [B,H,W,bp] with b real channels.  Returns the joined output bf16 [B,H,W,J] (J = 2b rounded up to a multiple of 8), or
    with ``split`` its two halves (P', Q') = (out[..., :b], out[..., b:2b]), each [B,H,W,bp]; pad channels are 0."""
    _chk_act(u, "u")
    _chk_act(c3, "c3")
    if tuple(u.shape) != tuple(c3.shape):
        raise ValueError(f"shufflev2_tail_fwd: u {tuple(u.shape)} and c3 {tuple(c3.shape)} differ")
    bp = c3.shape[-1]
    rows = c3.numel() // bp
    if split:
        y0, y1 = torch.empty_like(c3), torch.empty_like(c3)
    else:
        y0, y1 = torch.empty(*c3.shape[:-1], _v2_pitch(b), dtype=BF16, device=c3.device), None
    with _span("shufflev2_tail_fwd", 0.0, u, c3, y0, y1):
        _call("shufflev2_tail_fwd", _p(u), None if co_u is None else _p(co_u.scale), None if co_u is None else _p(co_u.shift),
              _p(c3), _p(co.scale), _p(co.shift), _p(y0), _p(y1), rows, b, bp)
    return (y0, y1) if split else y0


def shufflev2_tail_bwd(g, c3, co, b, cu=None, co_u=None):
    """Backward of shufflev2_tail_fwd for g = dL/dout: the joined gradient bf16 [B,H,W,J], or a pair (dL/dP', dL/dQ') of
    [B,H,W,bp].  Returns (dz3, partial3, du, partial_u): dz3 = dL/dv * [c3 * scale + shift > 0] bf16 [B,H,W,bp] with
    partial3 fp32 [T,2,bp] = {sum dz3, sum dz3 * c3}; du = dL/du (passthrough, partial_u None), or with ``cu`` / ``co_u``
    du = dL/du * [cu * scale + shift > 0] and partial_u = {sum du, sum du * cu}."""
    _chk_act(c3, "c3")
    bp = c3.shape[-1]
    rows = c3.numel() // bp
    g0, g1 = g if isinstance(g, (tuple, list)) else (g, None)
    _chk_act(g0, "g")
    if g1 is not None:
        _chk_act(g1, "g")
        if tuple(g0.shape) != tuple(c3.shape) or tuple(g1.shape) != tuple(c3.shape):
            raise ValueError(f"shufflev2_tail_bwd: split g {tuple(g0.shape)} / {tuple(g1.shape)} must be shaped like c3 "
                             f"{tuple(c3.shape)}")
    elif tuple(g0.shape) != (*c3.shape[:-1], _v2_pitch(b)):
        raise ValueError(f"shufflev2_tail_bwd: joined g {tuple(g0.shape)} does not match c3 {tuple(c3.shape)} at b={b}")
    if (cu is None) != (co_u is None):
        raise ValueError("shufflev2_tail_bwd: give cu and co_u together")
    if cu is not None:
        _chk_act(cu, "cu")
        if tuple(cu.shape) != tuple(c3.shape):
            raise ValueError(f"shufflev2_tail_bwd: cu {tuple(cu.shape)} must be shaped like c3 {tuple(c3.shape)}")
    T = repvgg_partial_rows(rows, bp)
    dz3, du = torch.empty_like(c3), torch.empty_like(c3)
    part3 = torch.empty(T, 2, bp, dtype=F32, device=c3.device)
    partu = torch.empty(T, 2, bp, dtype=F32, device=c3.device) if cu is not None else None
    with _span("shufflev2_tail_bwd", 0.0, g0, g1, c3, cu, dz3, du):
        _call("shufflev2_tail_bwd", _p(g0), _p(g1), _p(c3), _p(co.scale), _p(co.shift), _p(dz3), _p(part3), _p(cu),
              None if co_u is None else _p(co_u.scale), None if co_u is None else _p(co_u.shift),
              _p(du), _p(partu), rows, b, bp)
    return dz3, part3, du, partu


# --------------------------------------------------------------------------------------------------------- MAE pieces
I32 = torch.int32


def mae_shuffle(keys):
    """fp32 keys [B, P] -> (ids int32 [B, P], slot int32 [B, P]): ids = keys.argsort(dim=1, stable=True), slot its inverse."""
    keys = keys.contiguous()
    B, P = keys.shape
    ids = torch.empty(B, P, dtype=I32, device=keys.device)
    slot = torch.empty(B, P, dtype=I32, device=keys.device)
    _call("mae_shuffle", _p(keys), _p(ids), _p(slot), B, P)
    return ids, slot


def mae_patchify(x, ids, p, Nm):
    """fp32 NCHW x -> (vis bf16 [B, P - Nm, p*p*C], tgt fp32 [B, Nm, p*p*C]): (p1, p2, c)-ordered patch vectors in shuffle order."""
    B, C, H, W = x.shape
    P = ids.shape[1]
    K = p * p * C
    vis = torch.empty(B, P - Nm, K, dtype=BF16, device=x.device)
    tgt = torch.empty(B, Nm, K, dtype=F32, device=x.device)
    with _span("mae_patchify", 0.0, x, vis, tgt):
        _call("mae_patchify", _p(x), _p(ids), _p(vis), _p(tgt), B, C, H, W, p, Nm)
    return vis, tgt


def mae_gather_rows(src, ids, s0, n, rows_per_sample, row_offset=0, out_dtype=F32):
    """[B, n, D] rows src[b * rows_per_sample + ids[b, s0 + j] + row_offset] of the fp32 row matrix src (rows_per_sample 0:
    one table shared by every sample)."""
    B, P = ids.shape
    D = src.shape[-1]
    out = torch.empty(B, n, D, dtype=out_dtype, device=src.device)
    _call("mae_gather_rows", _p(src), rows_per_sample, row_offset, _p(ids), B, P, s0, n, D, _p(out),
          1 if out_dtype == F32 else 0)
    return out


def mae_assemble_fwd(enc, mask_embed, dpos, slot, Nm):
    """Decoder input fp32 [B, P, D] in patch order from the encoder rows fp32 [B, P - Nm, D] (shuffle order), the mask token
    and the decoder position table fp32 [P, D]."""
    B, P = slot.shape
    D = enc.shape[-1]
    dec = torch.empty(B, P, D, dtype=F32, device=enc.device)
    with _span("mae_assemble_fwd", 0.0, enc, dec):
        _call("mae_assemble_fwd", _p(enc), _p(mask_embed), _p(dpos), _p(slot), _p(dec), B, P, Nm, D)
    return dec


def mae_assemble_bwd(g, slot, Nm, d_dpos=None):
    """g bf16 [B, P, D] (gradient of the decoder input) -> (encoder-row gradient bf16 [B, P - Nm, D], d_dpos fp32 [P, D])."""
    B, P = slot.shape
    D = g.shape[-1]
    g_enc = torch.empty(B, P - Nm, D, dtype=BF16, device=g.device)
    if d_dpos is None:
        d_dpos = torch.empty(P, D, dtype=F32, device=g.device)
    with _span("mae_assemble_bwd", 0.0, g, g_enc, d_dpos):
        _call("mae_assemble_bwd", _p(g), _p(slot), _p(g_enc), _p(d_dpos), B, P, Nm, D)
    return g_enc, d_dpos


def mae_pos_grad(g, slot, Nm, out=None):
    """Gradient fp32 [P + 1, D] of the encoder pos_embed from the encoder-input gradient bf16 [B, P - Nm, D]; row 0 is 0."""
    B, P = slot.shape
    D = g.shape[-1]
    if out is None:
        out = torch.empty(P + 1, D, dtype=F32, device=g.device)
    _call("mae_pos_grad", _p(g), _p(slot), _p(out), B, P, Nm, D)
    return out


def mae_scatter_masked(dh, slot, Nm):
    """bf16 [B, P, D]: the rows dh bf16 [B, Nm, D] at their masked patch, zero elsewhere."""
    B, P = slot.shape
    D = dh.shape[-1]
    g = torch.empty(B, P, D, dtype=BF16, device=dh.device)
    with _span("mae_scatter_masked", 0.0, dh, g):
        _call("mae_scatter_masked", _p(dh), _p(slot), _p(g), B, P, Nm, D)
    return g


def mae_mse(pred, target, loss_scale=1.0):
    """(loss fp32 [1] = mean((pred - target)^2), gradient bf16 of pred = loss_scale * 2 (pred - target) / numel).
    loss_scale multiplies the gradient only (1 / accumulation steps), as in softmax_xent."""
    if pred.shape != target.shape or pred.dtype != F32 or target.dtype != F32:
        raise ValueError("mae_mse: pred and target must be fp32 tensors of one shape")
    pred, target = pred.contiguous(), target.contiguous()
    n = pred.numel()
    grad = torch.empty(pred.shape, dtype=BF16, device=pred.device)
    partial = torch.empty(_query("mae_mse_blocks"), dtype=F32, device=pred.device)
    loss = torch.empty(1, dtype=F32, device=pred.device)
    with _span("mae_mse", 3.0 * n, pred, target, grad):
        _call("mae_mse", _p(pred), _p(target), n, 2.0 * float(loss_scale) / n, _p(grad), _p(partial), _p(loss))
    return loss, grad


# --------------------------------------------------------------------------------------------------------- SupCon pieces
def supcon_max_dim():
    """Widest embedding row the SupCon loss kernels take."""
    return _query("supcon_max_dim")


def _supcon_rows(t, name, max_dim):
    if t.dim() != 2 or t.dtype != F32:
        raise ValueError(f"{name}: expected an fp32 [N, D] tensor, got {t.dtype} {tuple(t.shape)}")
    N, D = t.shape
    if D % 4 or D > max_dim:
        raise NotImplementedError(f"{name}: rows of width {D}; the SupCon kernels take widths that are multiples of 4 up to "
                                  f"{max_dim}")
    if not t.is_cuda:
        raise ValueError(f"{name}: expected a CUDA tensor, got one on {t.device}")
    return t.contiguous(), N, D


def supcon_normalize(z):
    """(e fp32 [N, D] = F.normalize(z, dim=1), norms fp32 [N]) of fp32 rows z [N, D]."""
    z, N, D = _supcon_rows(z, "supcon_normalize", 1 << 16)
    e = torch.empty_like(z)
    nrm = torch.empty(N, dtype=F32, device=z.device)
    with _span("supcon_normalize", 3.0 * N * D, z, e):
        _call("supcon_normalize_fwd", _p(z), _p(e), _p(nrm), N, D)
    return e, nrm


def supcon_normalize_bwd(de, e, nrm):
    """bf16 gradient [N, D] of the rows z from the gradient de fp32 [N, D] of e = F.normalize(z, dim=1)."""
    de, N, D = _supcon_rows(de, "supcon_normalize_bwd", 1 << 16)
    if e.shape != de.shape or nrm.shape != (N,):
        raise ValueError("supcon_normalize_bwd: de, e [N, D] and norms [N] must match")
    dz = torch.empty(N, D, dtype=BF16, device=de.device)
    with _span("supcon_normalize_bwd", 4.0 * N * D, de, e, dz):
        _call("supcon_normalize_bwd", _p(de), _p(e.contiguous()), _p(nrm), _p(dz), N, D)
    return dz


def supcon_loss(e, labels, temperature, base_temperature):
    """SupCon loss over the fp32 rows e [N, D] with int32 row labels [N]: (loss fp32 [1], L fp32 [N], npos fp32 [N]); L and
    npos (the log-sum-exp and positive count of every anchor) are what supcon_loss_bwd needs."""
    e, N, D = _supcon_rows(e, "supcon_loss", supcon_max_dim())
    if labels.dtype != I32 or labels.shape != (N,) or not labels.is_contiguous():
        raise ValueError(f"supcon_loss: labels must be a contiguous int32 [{N}] tensor")
    L = torch.empty(N, dtype=F32, device=e.device)
    npos = torch.empty(N, dtype=F32, device=e.device)
    rows = torch.empty(N, dtype=F32, device=e.device)
    loss = torch.empty(1, dtype=F32, device=e.device)
    with _span("supcon_loss", 2.0 * N * N * D, e):
        _call("supcon_loss_fwd", _p(e), _p(labels), N, D, float(temperature), float(base_temperature), _p(L), _p(npos),
              _p(rows), _p(loss))
    return loss, L, npos


def supcon_loss_bwd(e, labels, L, npos, grad_out, temperature, base_temperature, grad_scale=1.0):
    """fp32 gradient [N, D] of grad_scale * grad_out * loss with respect to e; grad_out is a device scalar read by the
    kernel (no host synchronisation), L / npos come from supcon_loss."""
    e, N, D = _supcon_rows(e, "supcon_loss_bwd", supcon_max_dim())
    if grad_out.dtype != F32 or grad_out.numel() != 1 or not grad_out.is_cuda:
        raise ValueError("supcon_loss_bwd: grad_out must be a one-element CUDA fp32 tensor")
    de = torch.empty_like(e)
    with _span("supcon_loss_bwd", 4.0 * N * N * D, e, de):
        _call("supcon_loss_bwd", _p(e), _p(labels), _p(L), _p(npos), _p(grad_out.contiguous()), float(grad_scale), N, D,
              float(temperature), float(base_temperature), _p(de))
    return de


def relu_bwd(dy, y):
    """bf16 dy masked by the bf16 ReLU output y (dy where y > 0, else 0)."""
    _chk_act(dy, "relu_bwd dy")
    _chk_act(y, "relu_bwd y")
    if dy.shape != y.shape:
        raise ValueError("relu_bwd: dy and y must have one shape")
    dx = torch.empty_like(dy)
    _call("supcon_relu_bwd", _p(dy), _p(y), _p(dx), dy.numel())
    return dx
