"""CPU: every leaf of the overlap aligner's cases (aln_leaf_cases.py), walk for walk against the plain matrix, in slots
that held anything before, and the CIGAR text and breaking points formed from the walks.

The emulation (tests/emu, aln_core.cuh in its host flavour) aligns every pair of a case like the batch runtime does and
records each leaf (AlnLeafRec).  Every leaf must be a leaf by edlib's 1 MB rule; its operations region must be the
plain matrix's traceback (aln_oracle_nw on the sub-pair: the shape is a leaf, so the oracle traces that matrix
directly) behind its holes; its end score the sub-pair's distance, and for a split's child the optimum the split gave
it.  Each leaf is then run alone (emu_leaf) in a slot first filled with zeros, 0xFF, 0xA5, random bytes and another
leaf's leftovers: operations, score and every counter must not change.  The counters then show that each case reaches
the edges its name promises."""
import functools

import numpy as np
import pytest

import aln_leaf_cases as lc
from aln_cases import STRIPE
from emu_lib import EmuAligner
from oracle_lib import ops_to_cigar, oracle_align, oracle_breaking_points
from racon_gpu_b200.aligner import LEAF_COUNTERS, is_leaf

CASES = lc.cases()
RUNS = [r for runs in CASES.values() for r in runs]
HOLE = 0xFF


@pytest.fixture(scope="module")
def emu():
    return EmuAligner()


def oracle_ops(orc, q, t):
    """(ops, distance) of the plain matrix; empty sides are all deletions / all insertions"""
    if not q or not t:
        return np.full(len(q) + len(t), 2 if not q else 1, dtype=np.uint8), len(q) + len(t)
    return oracle_align(orc, q, t)


@functools.lru_cache(maxsize=None)
def _leaves(name):
    """Every leaf of the run: (record, q, t) of the sub-pair, the run's edit distances."""
    r = {x["name"]: x for x in RUNS}[name]
    recs, scores = lc.emu_leaves(EmuAligner(), r)
    out = []
    for x in recs:
        q, t = r["pairs"][int(x["aln"])]
        out.append((x, q[x["r0"]:x["r0"] + x["n"]], t[x["c0"]:x["c0"] + x["m"]]))
    return out, scores


def _record_failures(tag, got, want):
    diff = [k for k in ("band", "score") + LEAF_COUNTERS + ("cells", "ops_hash") if got[k] != want[k]]
    return [f"{tag}: " + ", ".join(f"{k} {int(got[k])} != {int(want[k])}" for k in diff)] if diff else []


def leaf_failures(emu, orc, x, q, t):
    """The plain-matrix checks of one leaf; returns (failures, its region)."""
    where = lc.where(x)
    bad = []
    n, m = len(q), len(t)
    if not is_leaf(n, m):
        bad.append(f"{where}: not a leaf by edlib's rule")
    region, rec = emu.leaf(q, t, int(x["band"]))
    bad += _record_failures(f"{where}: alone in a zeroed slot against the batch", rec, x)
    ops, dist = oracle_ops(orc, q, t)
    want = np.concatenate([np.full(n + m - ops.shape[0], HOLE, dtype=np.uint8), ops])
    if not (region == want).all():
        p = int(np.flatnonzero(region != want)[0])
        bad.append(f"{where}: ops region byte {p} = {region[p]}, the plain matrix's traceback has {want[p]} "
                   f"({ops.shape[0]} ops, band {int(x['band'])})")
    if int(x["score"]) != dist:
        bad.append(f"{where}: end score {int(x['score'])}, the plain matrix has {dist}")
    if not (int(x["top"]) & 1) and int(x["band"]) - 2 != dist:
        bad.append(f"{where}: a split's child with band {int(x['band'])}, but its optimum is {dist}")
    if lc.ops_hash(region) != int(x["ops_hash"]):
        bad.append(f"{where}: ops_hash {int(x['ops_hash']):#x}, the region hashes to {lc.ops_hash(region):#x}")
    return bad, region


@pytest.mark.parametrize("name", [r["name"] for r in RUNS])
def test_every_leaf_equals_the_plain_matrix(emu, oracle, name):
    leaves, scores = _leaves(name)
    bad = []
    for x, q, t in leaves:
        bad += leaf_failures(emu, oracle, x, q, t)[0]
        if int(x["top"]) & 1 and int(x["score"]) != scores[int(x["aln"])]:
            bad.append(f"{lc.where(x)}: a top-level leaf whose score is not the alignment's distance")
    assert bad == [], "\n".join(bad[:20])


def _other_leaf(leaves, x):
    """The leaf whose leftovers a slot holds before x: the run's largest other leaf, with a band unlike x's"""
    cand = [(int(y["n"]) * int(y["m"]), k) for k, (y, _, _) in enumerate(leaves)
            if (int(y["aln"]), int(y["r0"]), int(y["c0"])) != (int(x["aln"]), int(x["r0"]), int(x["c0"]))
            and y["n"] > 0 and y["m"] > 0]
    if not cand:
        return None
    y, q, t = leaves[max(cand)[1]]
    band = -1 if int(x["band"]) >= 0 else int(y["score"]) + 2
    return q, t, band


@pytest.mark.parametrize("name", [r["name"] for r in RUNS])
def test_every_leaf_is_independent_of_what_its_slot_held(emu, name):
    leaves, _ = _leaves(name)
    bad = []
    for k, (x, q, t) in enumerate(leaves):
        base, rec0 = emu.leaf(q, t, int(x["band"]))
        other = _other_leaf(leaves, x)
        for poison in EmuAligner.POISONS:
            if poison == "leftovers" and other is None:
                continue
            region, rec = emu.leaf(q, t, int(x["band"]), poison=poison, seed=1000 + k, other=other)
            tag = f"{lc.where(x)} in a slot of {poison}" + (f" (a {len(other[0])}x{len(other[1])} leaf, band {other[2]})"
                                                             if poison == "leftovers" else "")
            if not (region == base).all():
                p = int(np.flatnonzero(region != base)[0])
                bad.append(f"{tag}: ops region byte {p} = {region[p]}, {base[p]} in a zeroed slot")
            bad += _record_failures(tag, rec, rec0)
    assert bad == [], "\n".join(bad[:20])


def _tot(leaves, k, pred=lambda x: True):
    return sum(int(x[k]) for x, _, _ in leaves if pred(x))


def _path_touches_band_edge(ops, best):
    i = j = 0
    for op in ops:
        i += op != 2
        j += op != 1
        if abs(i - j) == best:
            return True
    return False


def _alignment_region(r, leaves, k):
    q, t = r["pairs"][k]
    region = np.full(len(q) + len(t), HOLE, dtype=np.uint8)
    for x, lq, lt in leaves:
        if int(x["aln"]) == k and len(lq) + len(lt):
            region[x["r0"] + x["c0"]:x["r0"] + x["c0"] + len(lq) + len(lt)] = EmuAligner().leaf(lq, lt, int(x["band"]))[0]
    return region


@pytest.mark.parametrize("case", list(CASES))
def test_case_reaches_its_leaf_edges(emu, oracle, case):
    runs = CASES[case]
    r = runs[0]
    leaves, _ = _leaves(r["name"])
    inner = lambda x: x["n"] > 0 and x["m"] > 0
    assert _tot(leaves, "diag_rounds") > 0 and _tot(leaves, "up_rounds") + _tot(leaves, "left_rounds") > 0
    if case == "rule_edges":
        tops = {(int(x["n"]), int(x["m"])) for x, _, _ in leaves if int(x["top"]) & 1}
        for B, m in lc.RULE_EDGES:
            assert (64 * B, m) in tops, (B, m)  # the widest leaf is traced directly
            assert (64 * B, m + 1) not in tops  # one column more splits
        split = {int(x["aln"]) for x, _, _ in leaves if not int(x["top"]) & 1}
        assert all(x["band"] >= 0 for x, _, _ in leaves if int(x["aln"]) in split)
        assert len(split) == len(lc.RULE_EDGES)
    if case == "tall_leaves":
        ns = {int(x["n"]) for x, _, _ in leaves}
        for k in (1, 2, 3):
            assert all(STRIPE * k + d in ns for d in (-64, -1, 0, 1, 63, 64))
        partial = [x for x, _, _ in leaves if ((int(x["n"]) + 63) // 64) % 32 and int(x["n"]) > STRIPE]
        assert partial and max(-(-int(x["n"]) // STRIPE) for x, _, _ in leaves) > 40
        assert _tot(leaves, "reload_block") > 1000 and _tot(leaves, "tail", lambda x: x["tail_kind"] == 1) > 0
    if case == "diagonal_runs":
        for k in ("full_runs", "reload_block", "reload_col"):
            total = _tot(leaves, k)
            assert total > 0, f"no leaf of {r['name']} counted {k}"
        assert _tot(leaves, "diag_ops") > _tot(leaves, "matches")
        runs_mm = []
        for x, q, t in leaves:
            ops = oracle_ops(oracle, q, t)[0]
            mm = np.flatnonzero(np.diff(np.concatenate([[0], (ops == 3).astype(np.int8), [0]])))
            runs_mm += list(mm[1::2] - mm[0::2])
        assert max(runs_mm) >= 40  # an all-mismatch diagonal longer than a window
        assert any(x["band"] >= 0 and x["full_runs"] > 0 for x, _, _ in leaves)
    if case == "borders":
        assert _tot(leaves, "border_lanes") > 0
        assert _tot(leaves, "tail", lambda x: inner(x) and x["tail_kind"] == 1) > 0
        assert _tot(leaves, "tail", lambda x: inner(x) and x["tail_kind"] == 2) > 0
        shapes = {(int(x["n"]), int(x["m"]), int(x["top"]) & 1) for x, _, _ in leaves}
        assert any(n == 1 for n, _, _ in shapes) and any(m == 1 for _, m, _ in shapes)
        assert any(n == 0 and top for n, _, top in shapes) and any(m == 0 and top for _, m, top in shapes)
        assert any(n == 0 and not top for n, _, top in shapes)  # children of r = -1 / r = n - 1
        splits = set()
        for k, (q, t) in enumerate(r["pairs"]):
            for s in emu.align_log(q, t, aln=k):
                splits.add("first" if s["r"] == -1 else "last" if s["r"] == s["n"] - 1 else "inner")
        assert {"first", "last"} <= splits, splits
    if case == "tight_bands":
        small = [(x, q, t) for x, q, t in leaves if not int(x["top"]) & 1 and int(x["score"]) <= 4]
        assert any(x["score"] == 0 and x["band"] == 2 for x, _, _ in small)
        assert any(x["score"] > 0 and _path_touches_band_edge(oracle_ops(oracle, q, t)[0], int(x["score"]))
                   for x, q, t in small)
    if case == "letters":
        other = lambda s: any(c not in b"ACGT" for c in s)
        assert any(other(t) and other(q) and inner(x) and not int(x["top"]) & 1 for x, q, t in leaves)
        assert any(other(t) and int(x["top"]) & 1 for x, q, t in leaves)
    if case == "guessed_top":
        tops = [x for x, _, _ in leaves if int(x["top"]) & 1]
        assert len(tops) == 3 and all(int(x["band"]) == -1 and int(x["top"]) == 1 for x in tops)
        for k in (3, 4):
            q, t = r["pairs"][k]
            from aln_cases import guess_of
            log = emu.align_log(q, t, guess=guess_of(len(q), len(t), r["permille"]), aln=k)
            assert log[0]["level"] == 0 and log[0]["band"] >= 0  # the split sub-problems do get the guess
        for k in range(3):  # a guess on a leaf-shaped top (the emulation's ALN_GUESS branch): no band, the same walk
            q, t = r["pairs"][k]
            g, _ = emu.align_leaves(q, t, guess=40, aln=k)
            assert g.shape[0] == 1 and int(g[0]["top"]) == 3 and int(g[0]["band"]) == -1
            assert _record_failures("guessed top", g[0], tops[k]) == []
    if case == "cigar_edges":
        cig = [ops_to_cigar(oracle, oracle_ops(oracle, q, t)[0]) for q, t in r["pairs"]]
        text = b" ".join(cig)
        for L in lc.DIGIT_EDGES:
            for letter in b"MID":
                assert f"{L}{chr(letter)}".encode() in text, (L, chr(letter))
        assert b"1M1I" * 32 in text
        holes = [(reg.shape[0] // 32 > 0 and (reg[:reg.shape[0] // 32 * 32].reshape(-1, 32) == HOLE).all(axis=1).any())
                 for reg in (_alignment_region(r, leaves, k) for k in range(3))]
        assert all(holes)
    if case == "bp_edges":
        assert {x["window_length"] for x in runs} == set(lc.BP_WINDOWS)
        seen = set()
        for x in runs:
            w = x["window_length"]
            for (q, t), (q_first, t_begin) in zip(x["pairs"], x["coords"]):
                seen.add(("start", t_begin % w == 0, t_begin % w == w - 1))
                ops = oracle_ops(oracle, q, t)[0]
                tpos = t_begin + np.cumsum(ops != 1) - (ops != 1)  # target coordinate each op is at
                n_win = (t_begin + len(t) - 1) // w - t_begin // w + 1
                seen.add(("windows>32", n_win > 32))
                cols = np.unique(tpos[(ops == 0) | (ops == 3)] // w)
                seen.add(("no match column", cols.shape[0] < n_win))
                # an insertion after the last column of a window (w > 1: with w = 1 every insertion is there)
                seen.add(("ins at end", bool(((ops == 1) & (tpos % w == 0) & (np.arange(len(ops)) > 0)).any() and w > 1)))
                d = ops == 2
                seen.add(("del across end", bool((d[1:] & d[:-1] & (tpos[1:] % w == 0)).any())))
                seen.add(("runs>32", int((np.diff(ops.astype(np.int16)) != 0).sum()) > 32))
        for want in [("start", True, False), ("windows>32", True), ("no match column", True), ("ins at end", True),
                     ("del across end", True), ("runs>32", True)]:
            assert want in seen, want
        assert any(k[0] == "start" and k[2] for k in seen)


def test_walk_counters_of_leaves_traced_by_hand(emu):
    """Walks short enough to follow by hand.  64 identical rows: a full run of 32 from the last cell, a reload by column
    (32 > 24 columns walked), a second full run whose last lane rates column 0.  96 identical rows: the first run ends at
    the block edge, so the window is reloaded for the block above.  One query character in front of 40: a full run, a
    reload by column, a run of 8 that stops at column 0, then a one-insertion tail."""
    rng = np.random.default_rng(1)
    s = lc.ACGT[rng.integers(0, 4, 96)].tobytes()
    t40 = b"C" + s[1:40]
    zero = dict(zip(LEAF_COUNTERS, [0] * len(LEAF_COUNTERS)))
    for q, t, want in ((s[:64], s[:64], dict(diag_rounds=2, diag_ops=64, matches=64, full_runs=2, reload_col=1, border_lanes=1)),
                       (s, s, dict(diag_rounds=3, diag_ops=96, matches=96, full_runs=3, reload_block=1, reload_col=1,
                                   border_lanes=1)),
                       (b"A" + t40, t40, dict(diag_rounds=2, diag_ops=40, matches=40, full_runs=1, reload_col=1,
                                              border_lanes=1, tail=1, tail_kind=1))):
        want = dict(zero, **want)
        for band in (-1, 2 + len(q) - len(t)):
            rec = emu.leaf(q, t, band)[1]
            got = {k: int(rec[k]) for k in LEAF_COUNTERS}
            diff = [f"{k} {got[k]} != {want[k]}" for k in LEAF_COUNTERS if got[k] != want[k]]
            assert diff == [], f"leaf r0=0 c0=0 {len(q)}x{len(t)} band {band}: " + ", ".join(diff)
            assert int(rec["score"]) == len(q) - len(t) and int(rec["cells"]) <= len(q) * len(t)


def test_the_ops_hash_sees_every_change(emu, oracle):
    """aln_ops_digest (C) equals its restatement, and flipping any one operation, turning one into a hole or swapping
    two different ones changes it."""
    leaves, _ = _leaves("diagonal_runs")
    rng = np.random.default_rng(5)
    for x, q, t in leaves[:4]:
        region, rec = emu.leaf(q, t, int(x["band"]))
        h = emu.ops_digest(region)
        assert h == int(rec["ops_hash"]) == lc.ops_hash(region)
        for p in range(region.shape[0]):
            for v in (0, 1, 2, 3, HOLE):
                if v != region[p]:
                    y = region.copy()
                    y[p] = v
                    assert lc.ops_hash(y) != h, (lc.where(x), p, v)
        for p, s in rng.integers(0, region.shape[0], size=(400, 2)):
            if region[p] != region[s]:
                y = region.copy()
                y[p], y[s] = region[s], region[p]
                assert lc.ops_hash(y) != h and emu.ops_digest(y) == lc.ops_hash(y), (lc.where(x), p, s)
        y = region.copy()
        y[-1] = HOLE
        assert emu.ops_digest(y) != h


@pytest.mark.parametrize("name", [r["name"] for r in CASES["cigar_edges"] + CASES["bp_edges"]])
def test_cigars_and_breaking_points_equal_the_oracle(emu, oracle, name):
    """The engine's CIGAR text (aln_cigar_text) and breaking points (aln_breaking_points) of the run, formed from its
    run starts, against the oracle's spelling of the plain matrix's operations and its restatement of racon."""
    r = {x["name"]: x for x in RUNS}[name]
    w = r["window_length"]
    for k, ((q, t), (q_first, t_begin)) in enumerate(zip(r["pairs"], r["coords"])):
        ops, dist = oracle_ops(oracle, q, t)
        got, score, _, _ = emu.align(q, t, q_first, t_begin, w)
        assert score == dist and (got == ops).all(), (name, k)
        assert emu.cigar == ops_to_cigar(oracle, ops), (name, k)
        if w:
            want = oracle_breaking_points(oracle, ops, q_first, t_begin, t_begin + len(t), w)
            assert emu.breaking_points.shape == want.shape and (emu.breaking_points == want).all(), (name, k)
