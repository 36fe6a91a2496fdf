"""The per-stream GEMM workspace cache (ops._workspace) stays out of CUDA-graph captures: a capture gets graph-private
scratch, so no later request that grows the cached buffer can free memory a captured graph still addresses."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_capture_gets_private_workspace_and_leaves_the_cache_alone():
    from deeplearning_b200 import ops

    dev = torch.device("cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        eager = ops._workspace(1 << 20, dev)
        assert ops._workspace(1 << 20, dev).data_ptr() == eager.data_ptr()   # eager calls share the cached buffer
    cached = {k: v.data_ptr() for k, v in ops._ws_cache.items()}
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        inside = ops._workspace(4 << 20, dev)
        assert inside.numel() >= 4 << 20 and inside.data_ptr() != eager.data_ptr()
    assert {k: v.data_ptr() for k, v in ops._ws_cache.items()} == cached
    with torch.cuda.stream(s):
        assert ops._workspace(1 << 20, dev).data_ptr() == eager.data_ptr()
