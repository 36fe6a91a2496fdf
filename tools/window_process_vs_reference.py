"""b200_window_partition / b200_window_merge against the REFERENCE's own CUDA extension swin_window_process compiled for sm_90a
(oracle/build_window_process_ref.py; SURVEY.md 2.3A beat-bar): bit-exact outputs and CUDA-event timings on the reference
unit-test shape (kernels/window_process/unit_test.py: B=192, 56x56x96, shift 2, window 7) and the Swin-T stage shapes at bs 128.
Prints a markdown table; python tools/window_process_vs_reference.py [output.md] also writes it to that file."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from deeplearning_b200.classification.swin_transformer.kernels.window_process.window_process import swin_window_process as ours
from oracle.build_window_process_ref import load_ref

ref = load_ref()
assert ref is not None, "build the reference extension first: python oracle/build_window_process_ref.py"


def timed(fn, reps=50):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


rows = []
for (B, H, C, shift, ws) in ((192, 56, 96, 2, 7), (128, 56, 96, 3, 7), (128, 28, 192, 3, 7), (128, 14, 384, 3, 7)):
    for dtype in (torch.float32, torch.float16):
        x = torch.randn(B, H, H, C, device="cuda").to(dtype)
        nW = (H // ws) ** 2
        for name, f_ref, f_ours, arg in (
            ("roll_and_window_partition_forward", ref.roll_and_window_partition_forward, ours.roll_and_window_partition_forward, x),
            ("roll_and_window_partition_backward", ref.roll_and_window_partition_backward, ours.roll_and_window_partition_backward,
             x.view(B * nW, ws, ws, C)),
            ("window_merge_and_roll_forward", ref.window_merge_and_roll_forward, ours.window_merge_and_roll_forward,
             x.view(B * nW, ws, ws, C)),
            ("window_merge_and_roll_backward", ref.window_merge_and_roll_backward, ours.window_merge_and_roll_backward, x),
        ):
            s = -shift if "partition_forward" in name or "roll_backward" in name else shift
            a = f_ref(arg, B, H, H, C, s, ws)
            b = f_ours(arg, B, H, H, C, s, ws)
            same = torch.equal(a.reshape(-1), b.reshape(-1))
            t_ref = timed(lambda: f_ref(arg, B, H, H, C, s, ws))
            t_ours = timed(lambda: f_ours(arg, B, H, H, C, s, ws))
            gb = 2 * x.numel() * x.element_size() / 1e9
            rows.append((f"{B}x{H}x{H}x{C}", str(dtype).replace("torch.", ""), name, same, t_ref, t_ours, gb / t_ref * 1e6, gb / t_ours * 1e6))
            assert same, (name, B, H, C, dtype)
out = ["| shape | dtype | function | bit-exact | reference .cu (us) | b200 (us) | reference GB/s | b200 GB/s | speed-up |", "|---|---|---|---|---|---|---|---|---|"]
for r in rows:
    out.append(f"| {r[0]} | {r[1]} | {r[2]} | {r[3]} | {r[4]:.1f} | {r[5]:.1f} | {r[6]:.0f} | {r[7]:.0f} | {r[4] / r[5]:.2f}x |")
text = "\n".join(out)
print(text)
if len(sys.argv) > 1:
    with open(sys.argv[1], "w") as f:
        f.write(text + "\n")
