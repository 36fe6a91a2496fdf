"""One launch path on each side of the C ABI.

C side: every kernel launch goes through ``B200_LAUNCH`` (csrc/host_utils.h), which launches with programmatic stream
serialization, counts the kernel for ``b200_launch_count()`` and checks the launch; the host helpers the entries share are
declared once in host_utils.h.  Python side: every library call goes through ``ops._call`` (launch entries: current stream,
error check naming the entry) or ``ops._query`` (sizing entries: a rejected shape raises with the library's message).

The source scans run anywhere; the query checks need only the built library; the launch-count checks compare the counter
with the library kernels ``torch.profiler`` records on an H100."""
import ast
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "deeplearning_b200")
CSRC = os.path.join(PKG, "csrc")


def _read(path):
    with open(path) as f:
        return f.read()


def _csrc(pattern):
    return sorted(n for n in os.listdir(CSRC) if re.fullmatch(pattern, n))


def test_csrc_launches_only_through_b200_launch():
    for name in _csrc(r".*\.cu"):
        assert "launch_pdl(" not in _read(os.path.join(CSRC, name)), f"{name} launches around B200_LAUNCH"
    for name in _csrc(r".*\.(cu|cuh|h)"):
        assert "B200_LAUNCHED" not in _read(os.path.join(CSRC, name)), name


def test_abi_files_share_the_host_helpers():
    helper_def = re.compile(r"\b(aligned16|opt16|as_stream|ew_blocks|ew_grid|grid_for|capped_grid)\s*\([^()]*\)\s*\{")
    for name in _csrc(r"abi_.*\.cu"):
        m = helper_def.search(_read(os.path.join(CSRC, name)))
        assert m is None, f"{name} defines its own {m.group(1)}; use the one in host_utils.h"


def _library_calls(tree):
    """(line, text) of every attribute b200_* and every _lib.check(...) in tree."""
    out = []
    for node in ast.walk(tree):
        if isinstance(node, ast.Attribute) and node.attr.startswith("b200_"):
            out.append((node.lineno, node.attr))
        if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "check"
                and isinstance(node.func.value, ast.Name) and node.func.value.id == "_lib"):
            out.append((node.lineno, "_lib.check"))
    return out


def test_python_calls_the_library_only_through_call_and_query():
    for dirpath, _, files in os.walk(PKG):
        for name in files:
            path = os.path.join(dirpath, name)
            if not name.endswith(".py") or path == os.path.join(PKG, "_lib.py"):
                continue
            tree = ast.parse(_read(path))
            if path == os.path.join(PKG, "ops.py"):
                tree.body = [n for n in tree.body if not (isinstance(n, ast.FunctionDef) and n.name in ("_call", "_query"))]
            calls = _library_calls(tree)
            assert not calls, f"{os.path.relpath(path, ROOT)} calls the library directly: {calls}"
    src = _read(os.path.join(PKG, "ops.py"))
    assert "_lib.check(" in src.split("\ndef _call(")[1].split("\ndef ")[0]


# (entry, arguments it rejects, the reason the library gives)
REJECTED_QUERIES = [
    ("bn_bwd_blocks", (100, 96), "C=96 must be 8*2^k <= 2048"),
    ("layernorm_bwd_blocks", (100, 2048), "C=2048 must be a multiple of 8 and <= 1024"),
    ("dw_partial_rows", (100, 12), "C a multiple of 8 in [8, 8192]"),
    ("repvgg_partial_rows", (0, 64), "rows must be >= 1"),
    ("vgg_pool_partial_rows", (2, 8, 8, 12), "C must be a multiple of 8 in [8, 8192]"),
    ("conv2d_grouped_fwd_stats_rows", (2, 8, 8, 96, 3, 3, 1), "C=96 must be a multiple of 64"),
    ("conv2d_grouped_wgrad_workspace_bytes", (2, 8, 8, 96, 3, 3, 1), "C=96 must be a multiple of 64"),
]


@pytest.mark.parametrize("sym,args,reason", REJECTED_QUERIES, ids=[q[0] for q in REJECTED_QUERIES])
def test_query_raises_with_the_library_reason(sym, args, reason):
    from deeplearning_b200 import _lib, ops

    lib = _lib.load()
    # leave a different message behind first: the query must set its own
    assert lib.b200_conv2d_fwd(None, None, None, 1, 8, 8, 64, 64, 5, 1, None, None, 0, None, None, 0, None, None, None) == -1
    with pytest.raises(RuntimeError) as e:
        ops._query(sym, *args)
    msg = str(e.value)
    assert f"b200_{sym}{args}" in msg and reason in msg, msg
    assert "ksize" not in msg, msg


def test_query_returns_the_value_unchanged():
    from deeplearning_b200 import _lib, ops

    lib = _lib.load()
    assert ops._query("bn_bwd_blocks", 256 * 56 * 56, 64) == lib.b200_bn_bwd_blocks(256 * 56 * 56, 64) > 0
    assert ops._query("conv2d_fwd_stats_rows", 256, 56, 56, 64, 3, 1) == 132 * 8
    assert ops._query("repvgg_partial_rows", 1000, 64) == lib.b200_repvgg_partial_rows(1000, 64) > 0
    assert ops._query("conv2d_wgrad_workspace_bytes", 256, 56, 56, 64, 64, 3, 1) == \
        lib.b200_conv2d_wgrad_workspace_bytes(256, 56, 56, 64, 64, 3, 1) > 0
    assert ops.repvgg_partial_rows(1000, 64) == lib.b200_repvgg_partial_rows(1000, 64)


@pytest.mark.gpu
def test_relu_mask_sum_rejects_an_unsupported_width():
    from deeplearning_b200 import ops

    g = torch.zeros(4, 96, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match=re.escape("b200_bn_bwd_blocks(4, 96)") + ".*C=96 must be 8"):
        ops.relu_mask_sum(g, g.clone())


def _counted_and_profiled(fn):
    """(launch_count() delta, library kernels torch.profiler records) over fn()."""
    from torch.profiler import ProfilerActivity, profile

    from deeplearning_b200 import ops

    fn()   # warm-up: module loads, allocations, one-time attribute setup
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        n0 = ops.launch_count()
        fn()
        torch.cuda.synchronize()
        n1 = ops.launch_count()
    names = [e.name for e in prof.events() if "b200::" in e.name]
    return n1 - n0, names


def _bf16(*shape):
    return torch.randn(*shape, device="cuda").to(torch.bfloat16)


def _co(C):
    from deeplearning_b200 import ops

    co = ops.BnCoeffs(C, "cuda")
    for v in (co.mean, co.invstd, co.scale, co.shift):
        v.copy_(torch.rand(C, device="cuda") + 0.5)
    return co


def _op_cases():
    from deeplearning_b200 import ops

    B, H, W, C, Cr = 2, 14, 14, 64, 16
    x, dd = _bf16(B, H, W, C), _bf16(B, H, W, C)
    co = _co(C)
    f32 = dict(dtype=torch.float32, device="cuda")
    s, pool, gate = torch.randn(B, C, **f32), torch.randn(B, C, **f32), torch.rand(B, C, **f32)
    hpre, w1, w2 = torch.randn(B, Cr, **f32), torch.randn(Cr, C, **f32), torch.randn(C, Cr, **f32)
    dy = _bf16(B, H, W, 128)
    return {
        "dw_wgrad": lambda: ops.dw_wgrad(dd, x, 3, 1, co=co),
        "dw_relu_wgrad": lambda: ops.dw_relu_wgrad(dd, x, 1, co),
        "excite_bwd": lambda: ops.excite_bwd(s, pool, hpre, gate, w1, w2),
        "conv2d_wgrad": lambda: ops.conv2d_wgrad(dy, x, 3, 1),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["dw_wgrad", "dw_relu_wgrad", "excite_bwd", "conv2d_wgrad"])
def test_launch_count_matches_profiled_kernels_per_op(op):
    counted, names = _counted_and_profiled(_op_cases()[op])
    assert counted >= 2 and counted == len(names), (counted, names)


def _efficientnet():
    from deeplearning_b200.classification.efficientNet.models import network

    return network.efficientnet_b0(num_classes=10), 64


def _resnet():
    from deeplearning_b200.classification.resnet.models import networks

    return networks.resnet18(num_classes=10), 64


@pytest.mark.gpu
@pytest.mark.parametrize("make", [_efficientnet, _resnet], ids=["efficientnet_b0", "resnet18"])
def test_launch_count_matches_profiled_kernels_per_train_step(make):
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    m, hw = make()
    step = TrainStep(m.cuda().train(), lr=0.01)
    x = torch.randn(4, 3, hw, hw, device="cuda")
    y = torch.randint(0, 10, (4,), device="cuda")
    counted, names = _counted_and_profiled(lambda: step.step_eager(x, y))
    assert counted > 50 and counted == len(names), (counted, len(names))
