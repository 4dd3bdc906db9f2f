#!/usr/bin/env python3
"""Condense an ncu_summary.py CSV of ONE whole-batch step into a JSON file -- per kernel family (bench.py's
`graph.layer_kernels()` names) the DRAM bytes and ncu time of its launches.
usage: ncu_traffic_json.py <summary.csv> <out.json> <workload> <batch> [first_row] [n_rows]   (rows select one step of the capture)"""
import csv
import json
import re
import sys

FAMILY = [  # ncu kernel name (regex) -> family name used by the engine (engine.cu kStepName / layer_kernel)
    (r"stem_tc_kernel", "conv_stem_nchw_tcgen05"),
    (r"conv_window_tc_kernel", "conv_window_tcgen05"),
    (r"conv_gather_tc_kernel", "conv_gather_tcgen05"),
    (r"conv_dw3x3_tma", "conv_dw3x3_tma_dp4a"),
    (r"conv_dw_kernel", "conv_dw_direct"),
    (r"gemm_i8_tcgen05_kernel<[^,]*, *[^,]*, *[^,]*, *[^,]*>.*igemm|conv_igemm", "conv_igemm_i8_tcgen05"),
    (r"gemm_i8_tcgen05_kernel", "gemm_i8_tcgen05"),
    (r"pool", "pool"),
    (r"pointwise|relu_same_scale", "pointwise"),
    (r"concat", "concat_requant"),
    (r"upsample", "upsample_nearest"),
    (r"byte_lut", "byte_lut"),
    (r"softmax", "softmax"),
    (r"nhwc_to_nchw", "nhwc_to_nchw"),
    (r"nchw_to_nhwc", "nchw_to_nhwc"),
    (r"conv_stem_kernel", "conv_stem_nchw_dp4a"),
    (r"conv_direct", "conv_direct_dp4a"),
]


def family(name):
    for rx, f in FAMILY:
        if re.search(rx, name):
            return f
    return name


def main(src, out, workload, batch, first=0, count=None):
    rows = list(csv.DictReader(open(src)))
    rows = rows[first:first + count] if count else rows[first:]
    fam, total = {}, 0.0
    for r in rows:
        f = fam.setdefault(family(r["kernel"]), {"launches_per_step": 0, "dram_bytes_per_step": 0.0, "ncu_time_us_per_step": 0.0})
        f["launches_per_step"] += 1
        f["dram_bytes_per_step"] += float(r["dram_rd"] or 0) + float(r["dram_wr"] or 0)
        f["ncu_time_us_per_step"] += float(r["time_us"] or 0)
        total += float(r["time_us"] or 0)
    for f in fam.values():
        f["ncu_share_of_step"] = f["ncu_time_us_per_step"] / total if total else None
    json.dump({"source": f"{src} rows {first}..{first + len(rows) - 1} (ncu --set full --clock-control none, one whole-batch step)",
               "workload": workload, "batch": int(batch), "families": fam}, open(out, "w"), indent=1)
    print(json.dumps({k: round(v["ncu_share_of_step"], 3) for k, v in fam.items()}))


if __name__ == "__main__":
    a = sys.argv
    main(a[1], a[2], a[3], a[4], int(a[5]) if len(a) > 5 else 0, int(a[6]) if len(a) > 6 else None)
