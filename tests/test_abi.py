"""The C-ABI boundary: libb200cls.so loads on a CPU-only box and exports every symbol include/b200cls.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b200cls.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_\w+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/b200cls.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in deeplearning_b200/_lib.py"
    assert set(_lib.SIGNATURES) == set(names)


def test_host_metadata_without_gpu():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    assert lib.b200_abi_version() == 3
    # pure host-side planners are usable without a device
    # BN statistics rows: (persistent CTAs / channel blocks) x 4 row quadrants (x2 when the warp pair alternates tiles);
    # without a device the planner assumes the 132 SMs of an H100 SXM; channel blocks are 64 or 128 wide
    assert lib.b200_conv2d_fwd_stats_rows(256, 56, 56, 64, 3, 1) == 132 * 8
    assert lib.b200_conv2d_fwd_stats_rows(256, 56, 56, 256, 1, 1) == 132 // 2 * 4
    assert lib.b200_conv2d_fwd_stats_rows(256, 7, 7, 2048, 1, 1) == 128 // 16 * 4
    assert lib.b200_conv2d_fwd_stats_rows(1, 8, 8, 64, 1, 1) == 8
    assert lib.b200_conv2d_wgrad_workspace_bytes(256, 56, 56, 64, 64, 3, 1) > 0
    assert lib.b200_bn_bwd_blocks(256 * 56 * 56, 64) > 0
    assert lib.b200_bn_bwd_blocks(100, 96) == -1  # unsupported channel count is reported, not guessed


def test_rejected_call_returns_einval_with_message():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    rc = lib.b200_conv2d_fwd(None, None, None, 1, 8, 8, 64, 64, 5, 1, None, None, 0, None, None, 0, None, None, None)
    assert rc == -1  # B200_EINVAL: 5x5 is not supported, and nothing was launched
    assert "ksize" in _lib.last_error()


def test_no_per_thread_setters():
    """Every option of a call travels as an argument: the header declares no b200_*_set_* entry that arms the next call."""
    assert [n for n in _declared() if "_set_" in n] == []


def test_epilogue_options_are_checked_before_launch():
    """Inconsistent epilogue options are rejected with B200_EINVAL and a message before any CUDA or driver call, so these
    run without a device (the fake pointers are never dereferenced)."""
    from deeplearning_b200 import _lib

    lib = _lib.load()
    fake = 256
    for scale, shift in [(fake, None), (None, fake)]:   # the folded BatchNorm needs both coefficient vectors
        rc = lib.b200_conv2d_fwd(None, None, None, 1, 8, 8, 64, 64, 1, 1, None, None, 0, None, None, 0, scale, shift, None)
        assert rc == -1 and "bn_scale" in _lib.last_error(), _lib.last_error()
    rc = lib.b200_conv2d_wgrad(None, None, None, None, 0, 1, 8, 8, 64, 64, 1, 1, 0, None, fake, None)
    assert rc == -1 and "bias_partial" in _lib.last_error(), _lib.last_error()
    mask = _lib.BnMask(fake, fake, fake, fake)
    rc = lib.b200_conv2d_dgrad(None, None, None, 1, 8, 8, 64, 64, 3, 2, None, mask, None)
    assert rc == -1 and "stride 1" in _lib.last_error(), _lib.last_error()
    rc = lib.b200_gemm_dual(None, 64, None, 64, None, None, None, 128, 72, mask, None)
    assert rc == -1 and "N % 64" in _lib.last_error(), _lib.last_error()


def test_missing_library_fails_loudly(monkeypatch):
    from deeplearning_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libb200cls.so")
    try:
        _lib.load()
    except RuntimeError as e:
        assert "no CPU" in str(e)
    else:
        raise AssertionError("load() must raise when the CUDA extension is missing")


def test_wgrad_split_plan_is_one_wave_and_bounded():
    """Split-K plan of the weight-gradient GEMM (abi_conv.cu: plan_wgrad_geom), read back through the workspace size:
    workspace = splits * Cout * taps * Cin * 4 bytes. The cost model must keep (output tiles x splits) within one or two
    waves of the 132 SMs of an H100 SXM (no third, mostly empty wave) and never ask for an absurd amount of fp32 partials."""
    from deeplearning_b200 import _lib

    lib = _lib.load()

    def splits(B, H, W, Cin, Cout, k, s):
        nbytes = lib.b200_conv2d_wgrad_workspace_bytes(B, H, W, Cin, Cout, k, s)
        unit = Cout * k * k * Cin * 4
        assert nbytes % unit == 0
        return nbytes // unit

    def tiles(Cin, Cout, taps, merged=False):
        bn = 64 if Cin <= 64 else (256 if -(-Cin // 256) * 48 < -(-Cin // 128) * 32 else 128)
        if merged:
            return -(-Cout // 128) * (taps * 64 // (256 if taps % 4 == 0 else 192))
        return -(-Cout // 128) * -(-Cin // bn) * taps

    cases = [  # B, H, W, Cin, Cout, k, s, merged-tap mode
        (256, 56, 56, 64, 64, 3, 1, True), (256, 28, 28, 128, 128, 3, 1, False), (256, 14, 14, 256, 256, 3, 1, False),
        (256, 7, 7, 512, 512, 3, 1, False), (256, 7, 7, 512, 2048, 1, 1, False), (256, 56, 56, 64, 256, 1, 1, False),
        (256 * 197, 1, 1, 768, 3072, 1, 1, False), (256 * 197, 1, 1, 3072, 768, 1, 1, False), (256 * 197, 1, 1, 768, 2304, 1, 1, False),
        (128 * 3136, 1, 1, 96, 384, 1, 1, False), (256, 1, 1, 2048, 1000, 1, 1, False)]
    for B, H, W, Cin, Cout, k, s, merged in cases:
        sp = splits(B, H, W, Cin, Cout, k, s)
        pixel_blocks = -(-(B * (H // s) * (W // s)) // 64)
        assert 1 <= sp <= max(1, pixel_blocks // 4), (B, H, W, Cin, Cout, k, sp)
        items = tiles(Cin, Cout, k * k, merged) * sp
        if tiles(Cin, Cout, k * k, merged) <= 132:
            assert items <= 2 * 132, ("more than two waves", B, H, W, Cin, Cout, k, sp, items)
        assert sp * Cout * k * k * Cin * 4 <= 256 << 20   # at most 256 MB of partials per layer
