"""Stage N synthetic windows, upload once, time a few launches of the POA kernel with CUDA events, and print the phase
cycle counters (B200POA_PHASE_TIMERS=1 in the environment) and the sub-phase cycle counters (a library built with
-DB200POA_SUBTIMERS=1 by scripts/build_variant.sh, selected with B200POA_LIB)."""
import argparse, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from racon_gpu_b200 import api
from racon_gpu_b200.windows import synth_windows

ap = argparse.ArgumentParser()
ap.add_argument("--windows", type=int, default=1776)
ap.add_argument("--banded", type=int, default=1)
ap.add_argument("--launches", type=int, default=2)
ap.add_argument("--length", type=int, default=500)
ap.add_argument("--depth", type=int, default=32)
ap.add_argument("--err", type=float, default=0.15)
ap.add_argument("--mem-gb", type=float, default=24.0)
ap.add_argument("--max-seq", type=int, default=1023)
args = ap.parse_args()
b = synth_windows(args.windows, args.length, args.depth, args.err, seed=12345)
pb = api.PoaBatch(max_gpu_mem=int(args.mem_gb * (1 << 30)), banded=bool(args.banded), max_sequence_size=args.max_seq)
n, _ = pb.add_windows(b)
assert n == args.windows
pb.upload()
torch.cuda.synchronize()
ms = []
for _ in range(args.launches):   # the batch runs on the legacy default stream here, torch's events see it
    a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    pb.launch()
    b_.record()
    torch.cuda.synchronize()
    ms.append(round(a.elapsed_time(b_), 2))
print("launch ms", ms, "windows/s", round(args.windows / (min(ms) / 1e3)))
pb.download()
cons, cov, st = pb.get_consensus()
print("windows", n, "failed", int((st != 0).sum()), "info", pb.info())
pc = pb.phase_cycles()
if pc:
    tot = sum(pc.values())
    print("phase cycles per window per launch:", {k: round(v / n / args.launches / 1e6, 2) for k, v in pc.items()}, "Mcycles; total", round(tot / n / args.launches / 1e6, 2))

try:
    import ctypes
    lib = ctypes.CDLL(os.environ.get("B200POA_LIB", os.path.join(ROOT, "racon_gpu_b200", "libb200poa.so")))
    f = lib.b200poa_debug_subtimers
    buf = (ctypes.c_ulonglong * 32)()
    f(buf)
    names = {0: "program.A", 1: "program.B", 2: "add.a", 3: "add.b", 4: "add.c", 5: "add.d", 6: "topsort.1", 7: "topsort.2a",
             8: "topsort.2b", 9: "topsort.3", 11: "traceback.steps", 12: "traceback.tile_load", 13: "consensus.scores",
             14: "consensus.branch_completion", 15: "consensus.emit"}
    print("sub-phase Mcycles per window per launch:", {names.get(i, i): round(buf[i] / n / args.launches / 1e6, 2) for i in range(32) if buf[i]})
except AttributeError:
    pass
