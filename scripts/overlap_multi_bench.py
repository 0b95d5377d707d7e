"""Times the overlap path with several workers and with split contigs (b200poa_polish_overlaps_multi) and prints one
JSON line.  The card's name and power limit are read in the same run; the variants of each comparison alternate.
  short_reads   scripts/deep_window_bench.py's workload (150-base reads, --coverage, second tier on) at devices=[0]
                against [0, 0]: one worker against two on one device;
  long_contig   one contig of --long-length bases with 10 kb reads at --long-coverage, unsplit (one aligner batch of
                --big-aligner-mem) against forced into units by --small-aligner-mem; outputs must be equal;
  all_devices   when more than one device is visible: devices=[] (one worker on each) against [0] on the long contig.
Usage: python scripts/overlap_multi_bench.py [--length 400000] [--coverage 100] [--long-length 2000000] [--repeat 2]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402


def timed(fn, variants, repeat):
    """variants: name -> kwargs; alternated, the first pass of each a warm-up.  Returns name -> (median ms, last result)"""
    ms = {k: [] for k in variants}
    last = {}
    for _ in range(repeat + 1):
        for k, kw in variants.items():
            t0 = time.perf_counter()
            last[k] = fn(**kw)
            ms[k].append((time.perf_counter() - t0) * 1e3)
    return {k: (float(np.median(v[1:])), last[k]) for k, v in ms.items()}


def same(a, b):
    return a[0] == b[0] and (a[1] == b[1]).all() and (a[2] == b[2]).all()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--length", type=int, default=400_000)
    ap.add_argument("--coverage", type=float, default=100.0)
    ap.add_argument("--long-length", type=int, default=2_000_000)
    ap.add_argument("--long-coverage", type=float, default=30.0)
    ap.add_argument("--big-aligner-mem", type=int, default=24 << 30)
    ap.add_argument("--small-aligner-mem", type=int, default=160 << 20)
    ap.add_argument("--repeat", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    from deep_window_bench import short_reads
    from racon_gpu_b200 import api
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().split("\n")[0]
    scores = {"match": 5, "mismatch": -4, "gap": -8}
    out = {"gpu": card, "repeat": args.repeat, "visible_devices": torch.cuda.device_count()}

    s = short_reads(args.length, args.coverage)
    kw = dict(window_length=500, quality_threshold=10.0, tgs=False, trim=True, mem_per_poa_batch=8 << 30,
              deep_windows=True, **scores)
    r = timed(lambda **v: api.polish_overlaps(**s, **kw, **v), {"one_worker": {"devices": [0]},
                                                                "two_workers": {"devices": [0, 0]}}, args.repeat)
    assert same(r["one_worker"][1], r["two_workers"][1]), "one and two workers differ"
    n_win = (args.length + 499) // 500
    out["short_reads"] = {
        "workload": f"{args.length} b contig, 150 b reads at {args.coverage:g}x: {len(s['t_id'])} overlaps, {n_win} windows",
        **{k: {"ms": v[0], "windows_per_s": n_win / (v[0] / 1e3), "units": v[1][3]["rounds"],
               "polished": int(v[1][1].sum())} for k, v in r.items()}}

    s = short_reads(args.long_length, args.long_coverage, read_len=10_000, error=0.03, chunk=1000)
    kw = dict(window_length=500, quality_threshold=10.0, tgs=True, trim=True, mem_per_poa_batch=4 << 30, **scores)
    variants = {"unsplit": {"devices": [0], "aligner_mem": args.big_aligner_mem},
                "split": {"devices": [0], "aligner_mem": args.small_aligner_mem}}
    if torch.cuda.device_count() > 1:
        variants["all_devices"] = {"devices": [], "aligner_mem": args.small_aligner_mem}
    r = timed(lambda **v: api.polish_overlaps(**s, **kw, **v), variants, args.repeat)
    for k in variants:
        assert same(r["unsplit"][1], r[k][1]), f"{k} differs from the unsplit run"
    n_win = (args.long_length + 499) // 500
    out["long_contig"] = {
        "workload": f"{args.long_length} b contig, 10 kb reads at {args.long_coverage:g}x: {len(s['t_id'])} overlaps, "
                    f"{n_win} windows",
        **{k: {"ms": v[0], "aligner_mem": variants[k]["aligner_mem"], "units": v[1][3]["rounds"],
               "split_contigs": v[1][3]["split_contigs"], "repeat_overlaps": v[1][3]["repeat_overlaps"],
               "polished": int(v[1][1].sum()), "h2d_bytes": v[1][3]["h2d_bytes"]} for k, v in r.items()}}
    if "all_devices" not in variants:
        out["long_contig"]["all_devices"] = "not measured: one device visible"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
