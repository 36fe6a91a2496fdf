"""Condense `ncu --page raw --csv` exports / launch lists into small markdown tables.
usage: python tools/summarize_ncu.py raw <in.csv> <out.md> | launches <in.csv> <out.md> | traffic <in.csv> <out.md> <model>
("traffic": launch list taken with gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum; also refreshes the
model's entry of profiles/roofline_traffic.json, which bench.py reads for roofline.traffic when it exists)"""
import json
import os
import collections
import csv
import sys

COLS = [("gpu__time_duration.sum", "us"), ("dram__bytes_read.sum", "read"), ("dram__bytes_write.sum", "write"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram%"),
        ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "hmma%"),
        ("sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active", "hmma_inst%"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps%"), ("launch__registers_per_thread", "regs"),
        ("lts__t_sector_hit_rate.pct", "L2hit%"), ("l1tex__t_sector_hit_rate.pct", "L1hit%")]


def _table(path):
    rows = list(csv.reader(open(path)))
    for i, r in enumerate(rows):
        if "Kernel Name" in r:
            return r, rows[i + 1], rows[i + 2:]
    raise SystemExit("no header in " + path)


def raw(inp, out):
    hdr, units, data = _table(inp)
    idx = {h: i for i, h in enumerate(hdr)}
    with open(out, "w") as f:
        f.write(f"# ncu --set full summary of `{inp}` (one row per captured launch, serialized, cold cache)\n\n")
        f.write("| kernel | grid | " + " | ".join(f"{n} [{units[idx[c]]}]" for c, n in COLS if c in idx) + " |\n")
        f.write("|---|---|" + "---|" * sum(c in idx for c, _ in COLS) + "\n")
        for r in data:
            if len(r) < len(hdr):
                continue
            name = r[idx["Kernel Name"]].split("(")[0].replace("void ", "")[:44]
            vals = []
            for c, _ in COLS:
                if c in idx:
                    v = r[idx[c]]
                    try:
                        v = f"{float(v):.3f}".rstrip("0").rstrip(".")
                    except ValueError:
                        pass
                    vals.append(v)
            f.write(f"| {name} | {r[idx['Grid Size']]} | " + " | ".join(vals) + " |\n")


def launches(inp, out):
    hdr, _, _ = _table(inp)
    rows = list(csv.reader(open(inp)))
    start = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    idx = {h: i for i, h in enumerate(hdr)}
    agg, tot = collections.OrderedDict(), 0.0
    for r in rows[start + 1:]:
        if len(r) < len(hdr):
            continue
        n = r[idx["Kernel Name"]].split("(")[0].replace("void ", "")[:60]
        v = float(r[idx["Metric Value"]])
        u = r[idx["Metric Unit"]]
        v = v / 1000 if u == "ns" else (v * 1000 if u == "ms" else v)
        a = agg.setdefault(n, [0, 0.0])
        a[0] += 1
        a[1] += v
        tot += v
    with open(out, "w") as f:
        f.write(f"# ncu launch list of one training step (`{inp}`; gpu__time_duration, serialized, cold cache: compare SHARES)\n\n")
        f.write("| kernel | launches | total ms | share |\n|---|---|---|---|\n")
        for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| {n} | {c} | {t / 1000:.3f} | {100 * t / tot:.1f}% |\n")
        f.write(f"| **total** | {sum(c for c, _ in agg.values())} | {tot / 1000:.3f} | 100% |\n")


_SCALE = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}

# bench.py span name -> ncu kernel names whose bytes belong to it (a span covers the kernels one C-ABI entry point launches)
_SPANS = {"wgrad_gemm": ("wgrad_gemm_kernel", "wgrad_reduce_rows_kernel", "wgrad_reduce_flat_kernel"),
          "bn_bwd_reduce": ("bn_bwd_reduce_kernel",), "bn_bwd_apply": ("bn_bwd_apply_kernel",),
          "bn_apply": ("bn_apply_kernel",), "attention_fwd": ("attn_fwd2_kernel",),
          "attention_bwd": ("attn_bwd_kernel", "attn_delta_kernel"),
          "window_attention_fwd": ("wattn_fwd_kernel",), "window_attention_bwd": ("wattn_bwd_kernel",),
          "layernorm_fwd": ("layernorm_fwd_kernel",), "layernorm_bwd": ("layernorm_bwd_kernel",),
          "dwconv7": ("dwconv7_tile_kernel", "dwconv7_kernel"), "dwconv7_wgrad": ("dwconv7_wgrad_tile_kernel",)}


def traffic(inp, out, model):
    rows = list(csv.reader(open(inp)))
    start = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    idx = {h: i for i, h in enumerate(rows[start])}
    launches_, order = {}, []
    for r in rows[start + 1:]:
        if len(r) < len(idx):
            continue
        lid = r[idx["ID"]]
        if lid not in launches_:
            name = r[idx["Kernel Name"]].split("(")[0].replace("void ", "").split("<")[0].strip()
            launches_[lid] = {"name": name.split("::")[-1]}
            order.append(lid)
        v = float(r[idx["Metric Value"]].replace(",", "")) * _SCALE.get(r[idx["Metric Unit"]], 1.0)
        launches_[lid][r[idx["Metric Name"]]] = v
    agg, seen_loss = collections.OrderedDict(), False
    for lid in order:
        L = launches_[lid]
        n = L["name"]
        if n == "softmax_xent_kernel":
            seen_loss = True
        if n == "conv1x1_stream_kernel":   # the streaming 1x1 kernel serves the same C-ABI spans as the implicit-GEMM kernel
            n = "conv_gemm_kernel"
        if n == "conv_gemm_kernel" and model == "resnet50":
            n = "conv_gemm_kernel (backward: dgrad)" if seen_loss else "conv_gemm_kernel (forward)"
        a = agg.setdefault(n, [0, 0.0, 0.0, 0.0])
        a[0] += 1
        a[1] += L.get("gpu__time_duration.sum", 0.0)
        a[2] += L.get("dram__bytes_read.sum", 0.0)
        a[3] += L.get("dram__bytes_write.sum", 0.0)
    tot = sum(a[1] for a in agg.values())
    with open(out, "w") as f:
        f.write(f"# ncu launch list of one {model} training step (`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,"
                "dram__bytes_write.sum --clock-control none`, serialized, cold cache: compare SHARES)\n\n")
        f.write("| kernel | launches | total ms | share | DRAM read MB | DRAM write MB | DRAM GB/s |\n|---|---|---|---|---|---|---|\n")
        for n, (c, t, rd, wr) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| {n} | {c} | {t / 1000:.3f} | {100 * t / tot:.1f}% | {rd / 1e6:.0f} | {wr / 1e6:.0f} | "
                    f"{(rd + wr) / t / 1e3 if t else 0:.0f} |\n")
        f.write(f"| **total** | {sum(a[0] for a in agg.values())} | {tot / 1000:.3f} | 100% | "
                f"{sum(a[2] for a in agg.values()) / 1e6:.0f} | {sum(a[3] for a in agg.values()) / 1e6:.0f} | |\n")
    # bytes per launch of every bench.py span
    per = {}
    spans = dict(_SPANS)
    if model == "resnet50":
        spans["conv_gemm_fwd"] = ("conv_gemm_kernel (forward)",)
        spans["conv_gemm_dgrad"] = ("conv_gemm_kernel (backward: dgrad)",)
    else:
        spans["conv_gemm_fwd"] = ("conv_gemm_kernel",)
    for span, names in spans.items():
        hit = [agg[n] for n in names if n in agg]
        if hit and hit[0][0]:
            per[span] = sum(a[2] + a[3] for a in hit) / hit[0][0]
    tpath = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "roofline_traffic.json")
    allm = json.load(open(tpath)) if os.path.exists(tpath) else {}
    allm = {k: v for k, v in allm.items() if isinstance(v, dict)}
    allm[model] = per
    allm["_note"] = {"what": "DRAM bytes per launch (dram__bytes_read.sum + dram__bytes_write.sum, averaged over the launches of "
                             "one training step) for every bench.py kernel span, per model; wgrad_gemm includes its reduce pass",
                     "source": "tools/summarize_ncu.py traffic on an ncu launch list"}
    json.dump(allm, open(tpath, "w"), indent=1)


if __name__ == "__main__":
    {"raw": raw, "launches": launches, "traffic": traffic}[sys.argv[1]](*sys.argv[2:])
