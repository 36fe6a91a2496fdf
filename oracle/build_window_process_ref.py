"""TEST / BASELINE INFRASTRUCTURE - builds the REFERENCE's own CUDA extension `swin_window_process`
(classification/swin_transformer/kernels/window_process/swin_window_process{.cpp,_kernel.cu}, the only first-party CUDA of
the reference) for sm_90a, as the beat-this baseline of b200_window_partition / b200_window_merge (SURVEY.md 2.3A).

The sources are compiled from a scratch copy under /tmp (the reference tree is read-only and must not be copied into the
repo); the only edit is the one torch 2.x forces: `AT_DISPATCH_*(x.type(), ...)` -> `x.scalar_type()` (the implicit
DeprecatedTypeProperties -> ScalarType conversion was removed; the kernels are untouched).  Output: oracle/_ref/window_process/
swin_window_process_ref.so (git-ignored).  Run where the reference checkout is present: python oracle/build_window_process_ref.py
"""
import os
import re
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/classification/swin_transformer/kernels/window_process"
OUT = os.path.join(HERE, "_ref", "window_process")


def build():
    if not os.path.isdir(SRC):
        return os.path.exists(os.path.join(OUT, "swin_window_process_ref.so"))
    from torch.utils.cpp_extension import load

    tmp = "/tmp/swin_window_process_src"
    shutil.rmtree(tmp, ignore_errors=True)
    os.makedirs(tmp)
    for f in ("swin_window_process.cpp", "swin_window_process_kernel.cu"):
        text = open(os.path.join(SRC, f)).read()
        text = re.sub(r"(AT_DISPATCH_[A-Z_]+\(\s*\w+)\.type\(\)", r"\1.scalar_type()", text)
        open(os.path.join(tmp, f), "w").write(text)
    os.makedirs(OUT, exist_ok=True)
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    load(name="swin_window_process_ref", sources=[os.path.join(tmp, "swin_window_process.cpp"), os.path.join(tmp, "swin_window_process_kernel.cu")],
         build_directory=OUT, extra_cuda_cflags=["-O3"], is_python_module=True, verbose=False)
    return True


def load_ref():
    """Import the built extension (None when it has not been built)."""
    so = os.path.join(OUT, "swin_window_process_ref.so")
    if not os.path.exists(so):
        return None
    import importlib.util

    import torch  # noqa: F401  (the extension links against libtorch)

    spec = importlib.util.spec_from_file_location("swin_window_process_ref", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print("built" if build() else "reference checkout not present")
