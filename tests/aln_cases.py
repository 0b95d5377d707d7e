"""The overlap aligner's Hirschberg splits at their edges: batches of pairs, what the emulation says about each, and a
runner for the GPU side.

Every case is a list of runs (one batch configuration over a list of pairs).  The CPU suite runs every run's
top-level sub-problems through the emulation's split (tests/emu: one warp, and a team block on threads under the
protocol checker) and holds the middle columns against the plain distance matrix (tests/test_aln_splits.py).  The GPU
suite aligns the same batches on the digest build and compares the device's split log with the emulation's records,
split for split (tests/test_gpu_aln_splits.py).

`python aln_cases.py IN OUT` is the GPU worker: it runs the jobs pickled in IN on the library named by B200POA_LIB
(api.load_library() loads one library per process, so the digest build runs in a process of its own) and pickles the
results to OUT.
"""
from __future__ import annotations

import functools
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if _p not in sys.path:
        sys.path.insert(0, _p)

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
STRIPE = 64 * 32  # rows of one 32-block stripe
MB = 1 << 20


def run(name, pairs, permille=0, mem=8 << 30, rounds=1, paths=(), no_teams=False, more_items_than_blocks=False):
    """One batch: pairs [(q, t)], the band guess (b200aln_batch_set_band_guess: 0 never, > 0 fixed, -1 learnt from the
    previous round), the memory budget, align_all rounds on the same batch, the paths the split log must show."""
    return {"name": name, "pairs": pairs, "permille": permille, "mem": mem, "rounds": rounds, "paths": tuple(paths),
            "no_teams": no_teams, "more_items_than_blocks": more_items_than_blocks}


# ------------------------------------------------------------------------------------------------------------------
# pair builders
# ------------------------------------------------------------------------------------------------------------------
def _rand(rng, n):
    return rng.choice(ACGT, size=n).tobytes()


def mutated(rng, n, m, err):
    """A random target of m bases and a query of n bases derived from it with substitutions, insertions and deletions
    at rate err (cut or padded to exactly n)."""
    t = rng.choice(ACGT, size=m)
    out = []
    i = 0
    while i < m:
        x = rng.random()
        if x < err / 3:
            out.append(rng.choice(ACGT))
            i += 1
        elif x < 2 * err / 3:
            out.append(rng.choice(ACGT))
        elif x < err:
            i += 1
        else:
            out.append(t[i])
            i += 1
    q = np.asarray(out, dtype=np.uint8)[:n]
    if q.shape[0] < n:
        q = np.concatenate([q, rng.choice(ACGT, size=n - q.shape[0])])
    return q.tobytes(), t.tobytes()


def substituted(rng, n, k):
    """A target of n bases and the same with k substitutions, evenly spread: edit distance k."""
    t = rng.choice(ACGT, size=n)
    q = t.copy()
    for p in np.linspace(n // (2 * k + 2), n - 1 - n // (2 * k + 2), k).astype(np.int64) if k else []:
        q[p] = ACGT[(int(np.flatnonzero(ACGT == q[p])[0]) + 1 + int(rng.integers(0, 3))) % 4]
    return q.tobytes(), t.tobytes()


def guess_of(n, m, permille):
    """The host's guess for a top-level sub-problem (b200aln_batch_align_all), -1 for none."""
    from racon_gpu_b200.aligner import is_leaf
    if permille <= 0 or is_leaf(n, m):
        return -1
    return min((max(n, m) * permille + 999) // 1000 + 32, 1 << 29)


def learnt_permille(pairs, scores):
    """What a batch learns from an align_all for its next one (b200aln_batch_sync): 1.25 x the rate 90 % stay under."""
    rates = sorted((s * 1000 + max(len(q), len(t)) - 1) // max(len(q), len(t)) for (q, t), s in zip(pairs, scores)
                   if max(len(q), len(t)) > 0)
    if len(pairs) < 8 or len(rates) < 8:
        return 0
    return min(1000, rates[len(rates) * 9 // 10] * 5 // 4 + 1)


def n_for_band_residue(lo, permille, residue):
    """The smallest n >= lo whose guessed band (guess + 2) is congruent to residue mod 16."""
    n = lo
    while (guess_of(n, n, permille) + 2) % 16 != residue % 16:
        n += 1
    return n


def with_letters(rng, q, t, every=29):
    qa, ta = bytearray(q), bytearray(t)
    for k in range(int(rng.integers(0, every)), len(qa), every):
        qa[k] = ord("N")
    for k in range(int(rng.integers(0, every)), len(ta), every + 4):
        ta[k] = ord("N") if k % 2 else ord("R")
    return bytes(qa), bytes(ta)


# ------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def cases():
    rng = np.random.default_rng(2027)
    out = {}
    # one stripe up to more stripes than a team has warps (the hand-over ring wraps), odd and even m (lh != rh)
    edge = []
    for k in range(1, 7):
        for d in (-64, -1, 0, 1, 63, 64):
            n = STRIPE * k + d
            edge.append(mutated(rng, n, n + (k + d) % 2, 0.04))
    out["stripe_edges"] = [run("stripe_edges_whole", edge, permille=0, paths=("team",)),
                           run("stripe_edges_banded", edge, permille=120, paths=("team",))]
    # the guessed band starting on, just before and just after a 16-column word
    words = []
    for lo in (4500, 6100, 8300):
        for res in (0, 15, 1):
            n = n_for_band_residue(lo, 60, res)
            words.append(mutated(rng, n, n - 3, 0.03))
    out["word_edges"] = [run("word_edges", words, permille=60, paths=("team",))]
    # near-identical pairs and tiny bands: lower stripes start at c_lo > 0 and take the anchor
    tiny = [substituted(rng, n, k) for n, k in ((5000, 3), (9000, 6), (12300, 9), (4200, 0))]
    out["tiny_bands"] = [run("tiny_bands", tiny, permille=1, paths=("team",))]
    # n >> m: a long insertion, so that the lower stripes' strips leave the matrix (ALN_INF); and leaf-shaped ones
    tall = []
    for n, m in ((12000, 4000), (9000, 3000), (10500, 2600)):
        q, t = mutated(rng, m, m, 0.02)
        a = m // 2
        tall.append((q[:a] + _rand(rng, n - m) + q[a:], t))
    tall += [(_rand(rng, 12000), _rand(rng, 40)), (_rand(rng, 9000), _rand(rng, 300))]
    out["tall_thin"] = [run("tall_thin", tall, permille=0, paths=("team",))]
    # guesses too small, score - 1, score and generous: the redo on one warp and on a thin level's team
    p = 20
    gs = []
    for n in (2000, 6000, 8400):
        g = guess_of(n, n, p)
        for k in (3 * g, g + 1, g, g // 3):
            gs.append(substituted(rng, n, k))
    out["guesses"] = [run("guesses", gs, permille=p, paths=("warp", "team"))]
    # letters outside ACGT on teams: the cold loop, has_other per warp, each warp's share of the code row
    let = [with_letters(rng, *mutated(rng, n, n + 5, 0.06)) for n in (4500, 7000, 9100)]
    out["letters"] = [run("letters", let, permille=0, paths=("team",)), run("letters_banded", let, permille=150, paths=("team",))]
    # huge sub-problems (>= 8192 rows, >= 32 M cells) in a saturated level beside one-warp work, guessed (one redone),
    # then the same huge pairs in a thin level
    huge = [mutated(rng, 9300, 9250, 0.05)]
    g = guess_of(8800, 8800, 30)
    huge.append(substituted(rng, 8800, g + 1))
    fill = [mutated(rng, int(rng.integers(2100, 2600)), int(rng.integers(2100, 2600)), 0.1) for _ in range(2200)]
    out["saturated"] = [run("saturated", fill[:1100] + huge + fill[1100:], permille=30, mem=16 << 30, paths=("warp", "side")),
                        run("huge_thin", huge, permille=30, paths=("team",))]
    # more team work items than team blocks (the cursor reuses the progress words), two rounds on one batch; and a
    # budget too small for any team block: the same pairs on one warp
    cur = [mutated(rng, n, n - 7, 0.08) for n in (4300, 4700, 5200, 5600, 6100, 6500, 7000, 7400, 7900, 8100)]
    out["cursor"] = [run("cursor", cur, permille=-1, mem=0, rounds=2, paths=("team",), more_items_than_blocks=True),
                     run("no_teams", cur, permille=-1, mem=0, rounds=2, paths=("warp",), no_teams=True)]
    return out


# ------------------------------------------------------------------------------------------------------------------
# the emulation's records
# ------------------------------------------------------------------------------------------------------------------
def emu_records(emu, r, round_permille=None):
    """Per round: the emulation's split records of every pair (aln = its index in the batch), and the scores."""
    out = []
    permille = r["permille"] if r["permille"] >= 0 else 0
    for rnd in range(r["rounds"]):
        recs, scores = [], []
        for k, (q, t) in enumerate(r["pairs"]):
            recs.append(emu.align_log(q, t, guess=guess_of(len(q), len(t), permille), aln=k))
            _, score, _, _ = emu.align(q, t)
            scores.append(score)
        out.append((np.concatenate(recs) if recs else recs, scores))
        if r["permille"] < 0:
            permille = learnt_permille(r["pairs"], scores)
    return out


KEY = ("aln", "r0", "c0", "n", "m", "attempt")
VALUES = ("band", "level", "r", "ls", "rs", "best", "lc_hash", "rr_hash")


def compare_logs(name, got, want) -> list:
    """Differences between the device's split log and the emulation's records, keyed by (aln, r0, c0, n, m, attempt):
    first the splits whose values differ (naming the alignment, the sub-problem and the path the device took), then
    the splits only one side has (the children of a wrong split)."""
    from racon_gpu_b200.aligner import SPLIT_PATHS
    bad = []
    g = {tuple(int(x[k]) for k in KEY): x for x in got}
    w = {tuple(int(x[k]) for k in KEY): x for x in want}
    if len(g) != len(got):
        bad.append(f"{name}: the device logged {len(got) - len(g)} splits twice")
    for key in sorted(set(g) & set(w)):
        diff = [k for k in VALUES if g[key][k] != w[key][k]]
        if diff:
            x, y = g[key], w[key]
            bad.append(f"{name}: alignment {key[0]} sub-problem r0={key[1]} c0={key[2]} {key[3]}x{key[4]} attempt {key[5]} "
                       f"on the path {SPLIT_PATHS[int(x['path'])]} (level {int(x['level'])}, band {int(x['band'])}): "
                       + ", ".join(f"{k} {x[k]:#x} != {y[k]:#x}" if k.endswith("hash") else f"{k} {int(x[k])} != {int(y[k])}"
                                   for k in diff))
    for key in sorted(set(w) - set(g))[:5]:
        bad.append(f"{name}: alignment {key[0]} sub-problem r0={key[1]} c0={key[2]} {key[3]}x{key[4]} attempt {key[5]}: "
                   "not in the device's log")
    for key in sorted(set(g) - set(w))[:5]:
        bad.append(f"{name}: alignment {key[0]} sub-problem r0={key[1]} c0={key[2]} {key[3]}x{key[4]} attempt {key[5]} "
                   f"({SPLIT_PATHS[int(g[key]['path'])]}): the emulation has no such split")
    return bad


# ------------------------------------------------------------------------------------------------------------------
# the GPU side
# ------------------------------------------------------------------------------------------------------------------
def gpu_runs(runs, digest: bool = True):
    """Run the batches in a process of their own on the digest build (or the product library).  Returns one dict per
    run: per round the edit distances, CIGARs and info, and on the digest build the split log."""
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


#: budgets tried, smallest first, for runs that need few or no team blocks (mem=0): from the smallest a batch accepts
#: (4 MB) up, a few slots' worth above what the pairs themselves take
SMALL_BUDGETS = [int(x * MB) for x in (4, 4.2, 4.5, 4.9, 5.4, 6, 7, 8.5, 10, 13, 17, 24, 32, 48)]


def _fits(r, info, logs):
    if not logs:
        return True
    if r["no_teams"]:
        return info["n_team_blocks"] == 0
    if r["more_items_than_blocks"]:
        nt = info["n_team_blocks"]
        if nt == 0:
            return False
        lv = [x["level"] for x in logs[0] if x["path"] == 1 and x["attempt"] == 0]
        return len(lv) > 0 and np.bincount(lv).max() > nt
    return True


def _gpu_job(r):
    from racon_gpu_b200.aligner import CUDABatchAligner
    budgets = SMALL_BUDGETS if r["mem"] == 0 else [r["mem"]]
    for mem in budgets:
        al = CUDABatchAligner(device_id=0, max_gpu_memory=mem)
        al.set_band_guess(r["permille"])
        rounds, logs, fits = [], [], True
        for rnd in range(r["rounds"]):
            k = 0
            for q, t in r["pairs"]:
                if not al.add_overlap(q, t):
                    break
                k += 1
            if k < len(r["pairs"]):
                fits = False
                break
            al.align_all()
            got = al.generate_cigar_strings()
            rounds.append({"cigars": [c for c, _ in got], "ed": [e for _, e in got], "info": al.info()})
            if r["digest"]:
                logs.append(al.split_log())
            al.reset()
        al.close()
        if fits and (not r["digest"] or _fits(r, rounds[0]["info"], logs)):
            return {"rounds": rounds, "logs": logs, "mem": mem}
    raise RuntimeError(f"{r['name']}: no budget gives the team blocks the case needs")


if __name__ == "__main__":
    with open(sys.argv[1], "rb") as fh:
        jobs = pickle.load(fh)
    results = [_gpu_job(r) for r in jobs]
    with open(sys.argv[2], "wb") as fh:
        pickle.dump(results, fh)
