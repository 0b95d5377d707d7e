"""The overlap aligner's leaves and output formation at their edges: batches of pairs, what the emulation says about
every leaf, and a runner for the GPU side.

A leaf (aln_core.cuh aln_leaf) stores its whole matrix as block records and walks back from the last cell; every
operation of every CIGAR is written there.  The CIGAR text and the breaking points are then formed from the run starts
(aln_runs, aln_cigar_text, aln_breaking_points).  Every case is a list of runs (one batch configuration over a list of
pairs).  The CPU suite holds every leaf of every run against the plain matrix and re-runs it in a slot filled with
garbage first (tests/test_aln_leaves.py); the GPU suite compares the digest build's leaf log with the emulation's
records, leaf for leaf, and the product library's outputs with the oracle's (tests/test_gpu_aln_leaves.py).

`python aln_leaf_cases.py IN OUT` is the GPU worker: it runs the jobs pickled in IN on the library named by
B200POA_LIB (api.load_library() loads one library per process) and pickles the results to OUT.
"""
from __future__ import annotations

import functools
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

from aln_cases import ACGT, STRIPE, _rand, mutated, substituted, with_letters

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

#: edlib's 1 MB rule at its edge: (blocks, the widest leaf of 64 x blocks rows), 20 B m + 8 m < 2^20 and not for m + 1
RULE_EDGES = ((1, 37449), (2, 21845), (31, 1669), (32, 1618), (33, 1569), (64, 814), (65, 801))
DIGIT_EDGES = (9, 10, 99, 100, 999, 1000, 9999, 10000)
BP_WINDOWS = (1, 7, 500)


def run(name, pairs, permille=0, window_length=0, coords=None):
    """One batch: pairs [(q, t)], the band guess (0 never, > 0 fixed), the window length for breaking points (0: none)
    and per pair (q_first, t_begin) (None: zeros)."""
    return {"name": name, "pairs": pairs, "permille": permille, "window_length": window_length,
            "coords": coords if coords is not None else [(0, 0)] * len(pairs)}


# ------------------------------------------------------------------------------------------------------------------
# pair builders
# ------------------------------------------------------------------------------------------------------------------
def _base_not(rng, *avoid):
    """A base none of `avoid` (bytes values or None)."""
    choices = [b for b in b"ACGT" if b not in avoid]
    return bytes([choices[int(rng.integers(0, len(choices)))]])


def _max_leaf_m(n):
    from racon_gpu_b200.aligner import is_leaf
    m = (1 << 20) // (20 * ((n + 63) // 64) + 8) + 1
    while not is_leaf(n, m):
        m -= 1
    return m


def _tall(rng, n, m):
    """n >> m: a mutated copy of the target somewhere inside random query rows."""
    qt, t = mutated(rng, m, m, 0.05)
    a = int(rng.integers(0, n - m + 1))
    return _rand(rng, a) + qt + _rand(rng, n - m - a), t


def _diagonal_runs(rng, L):
    """Exact stretches of L bases between single edits: an insertion in front of each, a deletion behind it, the
    stretch's first row at offsets 0, 1, 62 and 63 of a 64-row block."""
    q, t = bytearray(), bytearray()
    for o in (0, 1, 62, 63):
        while (len(q) + 1) % 64 != o % 64:  # matching bases up to the row before the insertion
            b = _rand(rng, 1)
            q += b
            t += b
        s = _rand(rng, L)
        q += _base_not(rng, q[-1] if q else None, s[0]) + s  # the inserted base cannot slide into its neighbours
        t += s
        t += _base_not(rng, s[-1])
        nxt = _base_not(rng, t[-1])
        q += nxt
        t += nxt
    tail = _rand(rng, 20)
    return bytes(q + tail), bytes(t + tail)


def _mismatch_diagonal(rng, L, flank=100):
    """Random flanks around L x 'C' against L x 'A': every path through the block pays L, the diagonal one is taken."""
    a, b = _rand(rng, flank), _rand(rng, flank)
    return a + b"C" * L + b, a + b"A" * L + b


def _split_r_minus1(rng, n):
    """The left half of the target is all deletions: the top-level split takes r = -1 (an n = 0 leaf)."""
    q = _base_not(rng, ord("A")) + _rand(rng, n - 1)
    return q, b"A" * n + q


def _split_r_last(rng, n):
    """The right half of the target is all deletions: the top-level split takes r = n - 1 (an n = 0 leaf)."""
    q = _rand(rng, n - 1) + _base_not(rng, ord("A"))
    return q, q + b"A" * n


def _m_runs(rng, lengths):
    """One M run of every length, separated by single insertions that cannot slide."""
    q, t = bytearray(), bytearray()
    for L in lengths:
        s = _rand(rng, L)
        if q:
            q += _base_not(rng, q[-1], s[0])
        q += s
        t += s
    return bytes(q), bytes(t)


def _indel_runs(rng, lengths, deletions):
    """One insertion (or deletion) run of 'T's of every length between random stretches without a 'T' at their ends."""
    q, t = bytearray(), bytearray()
    for L in lengths:
        s = _base_not(rng, ord("T")) + _rand(rng, 198) + _base_not(rng, ord("T"))
        q += s
        t += s
        (t if deletions else q).extend(b"T" * L)
    s = _base_not(rng, ord("T")) + _rand(rng, 99)
    return bytes(q + s), bytes(t + s)


def _alternating(rng, k, kind):
    """k alternating runs inside random flanks: 'mismatch' substitutes every other base (match / mismatch runs, all
    spelled M), 'insert' puts a base after every base (M / I runs)."""
    a, core, b = _rand(rng, 60), bytearray(_rand(rng, k)), _rand(rng, 60)
    if kind == "mismatch":
        q = bytearray(core)
        for p in range(0, k, 2):
            q[p:p + 1] = _base_not(rng, core[p])
        return a + bytes(q) + b, a + bytes(core) + b
    q = bytearray()
    for p in range(k):
        q.append(core[p])
        q += _base_not(rng, core[p], core[p + 1] if p + 1 < k else b[0])
    return a + bytes(q) + b, a + bytes(core) + b


def _bp_pair(rng, w, t_begin):
    """For window length w and a segment starting at t_begin: a deletion over two whole windows, a window end inside
    an insertion run and one inside a deletion run, random edits around them."""
    unit = max(w, 8)
    q, t = mutated(rng, 6 * unit, 6 * unit, 0.05)
    q, t = bytearray(q), bytearray(t)
    # an insertion run exactly at a window end: the run lies between target positions p - 1 and p, t_begin + p = 0 mod w
    p = 2 * unit - (t_begin + 2 * unit) % w
    ins = _rand(rng, 12)
    t_ins = bytes(t[:p])
    q_ins = bytes(q[:p]) + ins  # the query's prefix aligned to t[:p] (mutations shift it a little: only roughly there)
    # a deletion run across a window end, and a deletion over two whole windows
    mid_t = bytes(t[p:]) + _rand(rng, 2 * w + 16) + _rand(rng, 3 * unit)
    mid_q = bytes(q[p:]) + mid_t[-3 * unit:]
    return q_ins + mid_q, t_ins + mid_t


# ------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def cases():
    from racon_gpu_b200.aligner import is_leaf
    rng = np.random.default_rng(4242)
    out = {}
    # the 1 MB rule: the widest leaf of B blocks, then one column more (a split whose children are banded leaves)
    edge = []
    for B, m in RULE_EDGES:
        n = 64 * B
        assert is_leaf(n, m) and not is_leaf(n, m + 1), (B, m)
        edge += [mutated(rng, n, m, 0.1), mutated(rng, n, m + 1, 0.1)]
    out["rule_edges"] = [run("rule_edges", edge)]
    # multi-stripe leaves with a partial last stripe against narrow targets, and one of more than 40 stripes
    tall = []
    for k in (1, 2, 3):
        for d in (-64, -1, 0, 1, 63, 64):
            n = STRIPE * k + d
            tall.append(_tall(rng, n, min(int(rng.integers(40, 200)), _max_leaf_m(n))))
    tall.append(_tall(rng, 83000, 40))
    out["tall_leaves"] = [run("tall_leaves", tall)]
    # exact diagonal stretches around the 32-cell window, at both ends of a block; all-mismatch diagonals; the same
    # stretches once more inside a pair that splits (banded child leaves)
    diag = [_diagonal_runs(rng, L) for L in (31, 32, 33, 63, 64, 65)]
    diag += [_mismatch_diagonal(rng, 40), _mismatch_diagonal(rng, 70)]
    diag.append((b"".join(q for q, _ in diag), b"".join(t for _, t in diag)))
    out["diagonal_runs"] = [run("diagonal_runs", diag)]
    # walks that reach column 0 with rows left / row 0 with columns left, splits at r = -1 and r = n - 1 (n = 0 leaves),
    # empty and one-character sides
    t0, q0 = _rand(rng, 400), _rand(rng, 400)
    bord = [(_rand(rng, 100) + t0, t0), (q0, _rand(rng, 100) + q0), _split_r_minus1(rng, 2000), _split_r_last(rng, 2000),
            (b"", _rand(rng, 50)), (_rand(rng, 50), b""), (b"A", _rand(rng, 300)), (_rand(rng, 300), b"C"), (b"G", b"G"),
            (b"G", b"T"), mutated(rng, 1, 900, 0.0), mutated(rng, 700, 1, 0.0)]
    out["borders"] = [run("borders", bord)]
    # near-identical pairs: child leaves with band best + 2 for a small best; single indels push the path to |i - j| = best
    tight = [substituted(rng, n, k) for n, k in ((3000, 1), (4000, 2), (5200, 3), (6000, 0), (3500, 4))]
    for n in (2600, 4100, 5000):
        q, t = substituted(rng, n, 2)
        a, b = n // 3, 2 * n // 3
        tight.append((q[:a] + q[a + 1:b] + _base_not(rng, q[b - 1], q[b]) + q[b:], t))
    out["tight_bands"] = [run("tight_bands", tight)]
    # bytes outside ACGT inside leaves, top-level ones and children of splits
    let = [with_letters(rng, *mutated(rng, n, n + 5, 0.06), every=17) for n in (300, 900, 1500, 3000, 4500)]
    out["letters"] = [run("letters", let)]
    # a batch with a band guess: its top-level leaves run without a band (the guess is for split sub-problems only)
    gt = [mutated(rng, n, n + 3, 0.08) for n in (500, 1200, 1600)] + [mutated(rng, n, n - 2, 0.08) for n in (3000, 5000)]
    out["guessed_top"] = [run("guessed_top", gt, permille=50)]
    # CIGAR text: run lengths at every digit boundary, more than 32 same-letter run starts, M / I alternating rounds,
    # all-hole chunks of operations, all-I and all-D alignments
    cig = [_m_runs(rng, DIGIT_EDGES), _indel_runs(rng, DIGIT_EDGES, False), _indel_runs(rng, DIGIT_EDGES, True),
           _alternating(rng, 150, "mismatch"), _alternating(rng, 80, "insert"), (_rand(rng, 300), b""),
           (b"", _rand(rng, 300)), (_rand(rng, 10000), b""), (b"", _rand(rng, 999))]
    out["cigar_edges"] = [run("cigar_edges", cig)]
    # breaking points: window lengths 1, 7 and 500, segments starting on a multiple of the window length and one before
    bp = []
    for w in BP_WINDOWS:
        pairs, coords = [], []
        for k, t_begin in enumerate((5 * w, 5 * w - 1, 37 * w, 37 * w - 1)):
            pairs.append(_bp_pair(rng, w, t_begin))
            coords.append((100 + 7 * k, t_begin))
            pairs.append(mutated(rng, 2000 + 300 * k, 2100, 0.12))
            coords.append((3 * k, t_begin))
        if w == 500:  # more than 32 windows in one alignment
            pairs.append(mutated(rng, 17500, 17000, 0.1))
            coords.append((11, 1000))
        bp.append(run(f"bp_edges_w{w}", pairs, window_length=w, coords=coords))
    out["bp_edges"] = bp
    return out


def noise_pairs():
    """Larger, heavily edited pairs (about 30 % edits, 2 - 5 kb) for a round before the cases: their leaves leave records
    of other matrices in the slots."""
    rng = np.random.default_rng(99)
    return [mutated(rng, int(rng.integers(2000, 5000)), int(rng.integers(2000, 5000)), 0.3) for _ in range(24)]


# ------------------------------------------------------------------------------------------------------------------
# the emulation's records
# ------------------------------------------------------------------------------------------------------------------
def emu_leaves(emu, r):
    """The emulation's leaf records of every pair of a run (aln = its index in the batch) and the edit distances."""
    from aln_cases import guess_of
    recs, scores = [], []
    for k, (q, t) in enumerate(r["pairs"]):
        x, s = emu.align_leaves(q, t, guess=guess_of(len(q), len(t), r["permille"]), aln=k)
        recs.append(x)
        scores.append(s)
    return np.concatenate(recs), scores


def ops_hash(region: np.ndarray) -> int:
    """aln_core.cuh aln_ops_digest restated: the wrapping sum over positions p of mix64((p << 8 | op) + golden)."""
    with np.errstate(over="ignore"):
        x = (np.arange(region.shape[0], dtype=np.uint64) << np.uint64(8)) | region.astype(np.uint64)
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
        return int(x.sum(dtype=np.uint64))


KEY = ("aln", "r0", "c0", "n", "m")


def leaf_values():
    from racon_gpu_b200.aligner import LEAF_COUNTERS
    return ("band", "top", "score") + LEAF_COUNTERS + ("cells", "ops_hash")


def where(x) -> str:
    return f"alignment {int(x['aln'])} leaf r0={int(x['r0'])} c0={int(x['c0'])} {int(x['n'])}x{int(x['m'])}"


def compare_logs(name, got, want) -> list:
    """Differences between a device leaf log and the emulation's records, keyed by (aln, r0, c0, n, m): first the leaves
    whose values differ (naming the leaf and every field), then duplicates and the leaves only one side has."""
    bad = []
    g = {tuple(int(x[k]) for k in KEY): x for x in got}
    w = {tuple(int(x[k]) for k in KEY): x for x in want}
    if len(g) != len(got):
        bad.append(f"{name}: the device logged {len(got) - len(g)} leaves twice")
    for key in sorted(set(g) & set(w)):
        x, y = g[key], w[key]
        diff = [k for k in leaf_values() if x[k] != y[k]]
        if diff:
            bad.append(f"{name}: {where(x)} (band {int(y['band'])}): "
                       + ", ".join(f"{k} {int(x[k]):#x} != {int(y[k]):#x}" if k == "ops_hash" else f"{k} {int(x[k])} != {int(y[k])}"
                                   for k in diff))
    for key in sorted(set(w) - set(g))[:5]:
        bad.append(f"{name}: {where(w[key])}: not in the device's log")
    for key in sorted(set(g) - set(w))[:5]:
        bad.append(f"{name}: {where(g[key])}: the emulation has no such leaf")
    return bad


# ------------------------------------------------------------------------------------------------------------------
# the GPU side
# ------------------------------------------------------------------------------------------------------------------
def gpu_runs(runs, digest: bool = True):
    """Run the batches in a process of their own on the digest build (or the product library).  Digest build, per run:
    the results and leaf log of the batch, of the same batch object after a round of noise_pairs(), and of a fresh batch
    with the pairs in reverse order (leaf log mapped back to the forward indices).  Product library, per run and
    skip_cigars setting: edit distances, CIGARs, operations and breaking points."""
    from racon_gpu_b200 import build
    lib = build.DIGEST_LIB if digest else build.LIB
    if not os.path.exists(lib):
        raise RuntimeError(f"{lib} is missing: run __graft_entry__.build()")
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.pkl"), os.path.join(d, "out.pkl")
        with open(src, "wb") as fh:
            pickle.dump([dict(r, digest=digest) for r in runs], fh)
        env = dict(os.environ, B200POA_LIB=lib)
        subprocess.run([sys.executable, os.path.abspath(__file__), src, dst], env=env, check=True, cwd=ROOT)
        with open(dst, "rb") as fh:
            return pickle.load(fh)


def _align(al, r, order, skip=False):
    """One align_all of the run's pairs in `order` on batch `al`; results indexed like r['pairs']."""
    pairs = r["pairs"]
    for k in order:
        (q, t), (q_first, t_begin) = pairs[k], r["coords"][k]
        st = al.lib.b200aln_batch_add_overlap(al.h, q, len(q), t, len(t), q_first, t_begin)
        assert st == 0, (r["name"], k, st)
    al.align_all()
    pos = {k: i for i, k in enumerate(order)}
    res = {}
    if r["window_length"]:  # (b200aln_batch_sync: before the operations can be read)
        bps = al.breaking_points()
        res["bp"] = [bps[pos[k]] for k in range(len(pairs))]
    if not skip:
        got = al.generate_cigar_strings()
        res["cigars"] = [got[pos[k]][0] for k in range(len(pairs))]
        res["ed"] = [got[pos[k]][1] for k in range(len(pairs))]
    res["ops"] = [al.ops(pos[k]) for k in range(len(pairs))]
    res["info"] = al.info()
    if r["digest"]:
        log = al.leaf_log()
        log["aln"] = np.asarray(order, dtype=np.int32)[log["aln"]]
        res["log"] = log
    al.reset()
    return res


def _batch(r, skip=False):
    from racon_gpu_b200.aligner import CUDABatchAligner
    al = CUDABatchAligner(device_id=0, max_gpu_memory=2 << 30)
    al.set_band_guess(r["permille"])
    if r["window_length"]:
        al.set_window_length(r["window_length"], skip_cigars=skip)
    return al


def _gpu_job(r):
    fwd = list(range(len(r["pairs"])))
    if not r["digest"]:
        out = {}
        for skip in ((False, True) if r["window_length"] else (False,)):
            al = _batch(r, skip)
            out[skip] = _align(al, r, fwd, skip)
            al.close()
        return out
    al = _batch(r)
    plain = _align(al, r, fwd)
    noise = noise_pairs()
    _align(al, dict(r, pairs=noise, coords=[(0, 0)] * len(noise), digest=False), list(range(len(noise))))
    after = _align(al, r, fwd)
    al.close()
    al = _batch(r)
    rev = _align(al, r, fwd[::-1])
    al.close()
    return {"plain": plain, "after_noise": after, "reversed": rev}


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    with open(sys.argv[1], "rb") as fh:
        jobs = pickle.load(fh)
    results = [_gpu_job(r) for r in jobs]
    with open(sys.argv[2], "wb") as fh:
        pickle.dump(results, fh)
