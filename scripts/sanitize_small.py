"""Tiny run for compute-sanitizer that creates, uses and destroys every kind of batch once:
POA consensus batches (full-span and partial-span windows, both band modes), a POA batch with MSA output whose second
launch outgrows its pinned MSA buffer, direct-mode POA batches (a polisher over a page-locked arena), the racon adapter's
batches, an aligner batch whose slots grow between two align_all rounds, and an aligner pool."""
import sys, os
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from racon_gpu_b200 import api
from racon_gpu_b200.aligner import AlignerPool, CUDABatchAligner, pack_pairs
from racon_gpu_b200.windows import synth_windows
from common import partial_span_windows, random_pairs

for b in (partial_span_windows(n=6, length=300, depth=10), synth_windows(6, 300, 10, 0.1, seed=3)):
    for banded in (False, True):
        pb = api.PoaBatch(max_gpu_mem=1 << 30, banded=banded)
        pb.add_windows(b)
        pb.generate_poa()
        cons, cov, st = pb.get_consensus()
        pb.close()
        print(banded, [len(c) for c in cons], st.tolist())

# the pinned MSA buffer starts at 1 MiB: the second launch's rows (about 2 MB) make it grow
pb = api.PoaBatch(max_gpu_mem=1 << 30, output_mask=api.OUTPUT_CONSENSUS | api.OUTPUT_MSA)
for n, length, depth in ((2, 300, 5), (120, 300, 30)):
    pb.reset()
    pb.add_windows(synth_windows(n, length, depth, 0.1, seed=5))
    pb.generate_poa()
    msa, st = pb.get_msa()
    print("msa", sum(len(m) * len(m[0]) for m in msa if m), "bytes,", int((st == 0).sum()), "of", len(st), "windows")
pb.close()

w = synth_windows(8, 300, 10, 0.1, seed=7, with_quality=True)
arena = api.WindowArena.from_batch(w)
pol = api.Polisher(devices=[0], batches_per_device=2, mem_per_batch=1 << 30)
cons, clen, polished, st = pol.polish_arena(arena, max_windows_per_round=4)
pol.close()
arena.close()
print("direct", clen.tolist(), polished.tolist())
cons, clen, polished, st, _ = api.polish_windows(w, devices=[0], mem_per_batch=1 << 30, via_adapter=True)
print("adapter", clen.tolist(), polished.tolist())

# slots are sized for 16 k columns first, then re-made for 32 k
al = CUDABatchAligner(device_id=0, max_gpu_memory=2 << 30)
for seed, shapes in ((11, [(2000, 0.1)] * 2), (12, [(20000, 0.1)])):
    for q, t in random_pairs(seed, shapes):
        assert al.add_overlap(q, t)
    al.align_all()
    print("aligner", [ed for _, ed in al.generate_cigar_strings()])
    al.reset()
al.close()

pool = AlignerPool(devices=(0,), batches_per_device=2, max_gpu_memory_per_batch=1 << 30)
ed, _, _, _, _ = pool.align(*pack_pairs(random_pairs(13, [(500, 0.1)] * 8)))
pool.close()
print("pool", ed.tolist())
