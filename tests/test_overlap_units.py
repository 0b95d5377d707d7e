"""CPU: the overlap driver's work units (racon_gpu_b200/csrc/host/overlap_units.hpp) and the aligner batch's admission
rule they share with b200aln.cu (host/aln_admission.hpp), in their host build (tests/emu/emu_units.cpp).

Checked on seeded overlap sets and on racon's lambda overlap lists (tests/golden/lambda_layers.npz): every window of a
contig with overlaps is owned by exactly one unit, which holds exactly the overlaps whose window span meets it, in
racon's order; without splitting the units are the rounds of a plain restatement of the greedy whole-contig staging; and
the edges -- overlaps that start or end on a window boundary, one overlap in three or more units, a unit boundary next
to windows without layers, a short last window, and a window whose overlaps alone exceed the budget."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
W = 500
SUCCESS, GENERIC_ERROR, INVALID_ARGUMENT = 0, 10, 15  # include/b200poa.h


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_units") / "libunits_emu.so"
    subprocess.run(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", str(so), "-x", "c++",
                    os.path.join(HERE, "emu", "emu_units.cpp")], check=True)
    return C.CDLL(str(so))


def _p(a, ty):
    return a.ctypes.data_as(C.POINTER(ty))


def synth(seed, contig_lengths, depth=20, read_len=(300, 1500), w=W):
    """The columns the planner reads (lengths only), racon's order interleaving contigs.  Reads are the contig segment's
    length give or take 10 %; a quarter of the overlaps start or end exactly on a window boundary."""
    rng = np.random.default_rng(seed)
    t_off = np.concatenate([[0], np.cumsum(contig_lengths)]).astype(np.int64)
    rows = []
    for c, ln in enumerate(contig_lengths):
        if ln < 200 or c == 1:  # contig 1 gets no overlap
            continue
        for _ in range(depth * ln // 1000):
            tb = int(rng.integers(0, ln - 100))
            te = min(ln, tb + int(rng.integers(*read_len)))
            x = rng.random()
            if x < 0.125 and te // w * w > tb:
                te = te // w * w  # ends on a boundary: t_end = k * w
            elif x < 0.25:
                tb = tb // w * w  # starts on one
            rows.append((c, tb, te, int((te - tb) * rng.uniform(0.9, 1.1)), int(rng.integers(0, 50))))
    rows = [rows[i] for i in rng.permutation(len(rows))]
    return columns(t_off, rows)


def columns(t_off, rows):
    """rows: (t_id, t_begin, t_end, read segment length, q_first), in racon's order"""
    q_len = np.asarray([r[3] for r in rows], np.int64)
    return {"t_off": np.asarray(t_off, np.int64), "t_id": np.asarray([r[0] for r in rows], np.int32),
            "t_begin": np.asarray([r[1] for r in rows], np.int32), "t_end": np.asarray([r[2] for r in rows], np.int32),
            "q_off": np.concatenate([[0], np.cumsum(q_len)]).astype(np.int64),
            "q_first": np.asarray([r[4] for r in rows], np.int32)}


def lambda_columns(case):
    from test_layer_cut import lambda_overlaps
    ov = lambda_overlaps(case)
    length = max(o["t_begin"] + len(o["t"]) for o in ov) + 137  # the contig runs on past the last overlap
    return columns([0, length], [(0, o["t_begin"], o["t_begin"] + len(o["t"]), len(o["q"]), o["q_first"]) for o in ov])


def plan(lib, s, budget, split, w=W):
    """(status, units as (contig, win_lo, win_hi, overlaps, split), stats dict)"""
    n_ov = len(s["t_id"])
    cap = 4 * n_ov + 16
    units = np.zeros((cap, 6), np.int64)
    ovl = np.zeros(cap * 4, np.int64)
    stats = np.zeros(5, np.int64)
    st = lib.emu_plan_units(C.c_int64(len(s["t_off"]) - 1), _p(s["t_off"], C.c_int64), C.c_int64(n_ov),
                            _p(s["t_id"], C.c_int32), _p(s["t_begin"], C.c_int32), _p(s["t_end"], C.c_int32),
                            _p(s["q_off"], C.c_int64), _p(s["q_first"], C.c_int32), C.c_int32(w), C.c_int64(budget),
                            C.c_int32(int(split)), _p(units, C.c_int64), C.c_int64(cap), _p(ovl, C.c_int64),
                            C.c_int64(ovl.shape[0]), _p(stats, C.c_int64))
    assert st != -100
    info = dict(zip(("split_contigs", "repeat_overlaps", "unfit_contig", "units", "overlaps"), stats.tolist()))
    out = [(int(u[0]), int(u[1]), int(u[2]), ovl[u[3]:u[4]].tolist(), bool(u[5])) for u in units[:info["units"]]]
    return st, out, info


class Load:
    """the aligner batch's admission (emu_admit) on a batch that cuts layers"""

    def __init__(self, lib, s, budget, w=W):
        self.lib, self.s, self.budget, self.w = lib, s, budget, w
        self.state = np.zeros(3, np.int64)

    def copy(self):
        c = Load(self.lib, self.s, self.budget, self.w)
        c.state = self.state.copy()
        return c

    def add(self, k):
        s = self.s
        return self.lib.emu_admit(_p(self.state, C.c_int64), C.c_int64(self.budget), C.c_int32(self.w), C.c_int32(1),
                                  C.c_int32(int(s["q_off"][k + 1] - s["q_off"][k])),
                                  C.c_int32(int(s["t_end"][k] - s["t_begin"][k])), C.c_int32(int(s["t_begin"][k]))) == 0

    def add_all(self, ks):
        return all(self.add(k) for k in ks)


def first_windows(s, w=W):
    lens = np.diff(s["t_off"])
    return np.concatenate([[0], np.cumsum((lens + w - 1) // w)]).astype(np.int64)


def by_contig(s):
    """racon's order of each contig's overlaps"""
    out = [[] for _ in range(len(s["t_off"]) - 1)]
    for k, c in enumerate(s["t_id"].tolist()):
        out[c].append(k)
    return out


def todays_rounds(lib, s, budget, w=W):
    """The greedy staging of the whole-contig driver, restated: one aligner batch per round, contigs added whole in
    contig order until one does not fit; that one starts the next round, or is reported when it fails an empty batch.
    Returns (unfit contig or -1, rounds as (win_lo, win_hi, overlaps))."""
    fw, ks = first_windows(s, w), by_contig(s)
    rounds, c, n = [], 0, len(ks)
    while c < n:
        c0, load = c, Load(lib, s, budget, w)
        while c < n:
            trial = load.copy()
            if trial.add_all(ks[c]):
                load, c = trial, c + 1
                continue
            if c == c0:
                return c, rounds
            break
        with_ov = [x for x in range(c0, c) if ks[x]]
        if with_ov:
            rounds.append((int(fw[with_ov[0]]), int(fw[with_ov[-1] + 1]), [k for x in with_ov for k in ks[x]]))
    return -1, rounds


def min_budget(lib, s, ks, w=W):
    """the smallest aligner budget that takes the overlaps ks in one batch"""
    lo, hi = 1, 1 << 40
    while lo < hi:
        mid = (lo + hi) // 2
        if Load(lib, s, mid, w).add_all(ks):
            hi = mid
        else:
            lo = mid + 1
    return lo


def scaled_budget(lib, s, share, w=W):
    """the slots' share of a batch (what one short overlap needs) plus `share` of what the largest contig adds to it,
    and never less than what the overlaps of the fullest window need"""
    ks = by_contig(s)
    lo, hi = spans(s, w)
    fw = first_windows(s, w)
    largest = max(min_budget(lib, s, kc, w) for kc in ks if kc)
    base = min_budget(lib, s, [int(np.argmin(np.diff(s["q_off"])))], w)
    window = max(min_budget(lib, s, [k for k in kc if lo[k] <= x <= hi[k]], w)
                 for c, kc in enumerate(ks) if kc for x in range(int(fw[c + 1] - fw[c])))
    return max(window, int(base + share * (largest - base))), largest


def spans(s, w=W):
    """each overlap's first and last window in its contig (the planner's view of an empty overlap: its first window)"""
    n_win = np.diff(first_windows(s, w))[s["t_id"]]
    lo = np.minimum(s["t_begin"] // w, n_win - 1)
    hi = np.minimum(np.maximum(s["t_begin"], s["t_end"] - 1) // w, n_win - 1)
    return lo, hi


def check_units(s, units, w=W):
    """every window of a contig with overlaps owned once; each unit's overlaps in racon's order, exactly those meeting
    its windows (a whole-contig unit: every overlap of its contigs)"""
    fw, ks = first_windows(s, w), by_contig(s)
    lo, hi = spans(s, w)
    owner = np.full(int(fw[-1]), -1)
    contig_of = np.repeat(np.arange(len(ks)), np.diff(fw))
    for i, (c, a, b, ov, split) in enumerate(units):
        assert a < b and (owner[a:b] == -1).all()
        owner[a:b] = i
        assert ov == sorted(ov, key=lambda k: (s["t_id"][k], k))  # racon's order
        if split:
            assert (contig_of[a:b] == c).all()
            local = (a - fw[c], b - fw[c])
            want = [k for k in ks[c] if lo[k] < local[1] and hi[k] >= local[0]]
            assert ov == want
        else:
            cs = sorted(set(contig_of[a:b].tolist()))
            assert ov == [k for x in cs for k in ks[x]] and a == fw[cs[0]] and b == fw[cs[-1] + 1]
    for c, kc in enumerate(ks):
        if kc:
            assert (owner[fw[c]:fw[c + 1]] >= 0).all(), c
    return owner


SEEDS = {31: (12000, 0, 3100, 2500, 9000), 32: (20000, 1800, 700, 15000), 33: (7000, 0, 350, 7100, 260, 5300)}


@pytest.mark.parametrize("seed", list(SEEDS))
@pytest.mark.parametrize("share", [1.0, 0.45, 0.2])
def test_units_own_every_window_once_with_its_overlaps(emu, seed, share):
    s = synth(seed, SEEDS[seed])
    budget, largest = scaled_budget(emu, s, share)
    st, units, info = plan(emu, s, budget, True)
    assert st == SUCCESS, info
    check_units(s, units)
    n_split = sum(u[4] for u in units)
    assert (n_split == 0) == (share == 1.0)
    assert info["split_contigs"] == len({u[0] for u in units if u[4]})
    assert info["repeat_overlaps"] == sum(len(u[3]) for u in units) - len(s["t_id"])
    if share < 1.0:
        assert info["repeat_overlaps"] > 0
    # every unit is one the aligner batch takes
    for u in units:
        assert Load(emu, s, budget).add_all(u[3])


@pytest.mark.parametrize("seed", list(SEEDS))
@pytest.mark.parametrize("share", [4.0, 1.3, 1.0, 0.5])
def test_unsplit_units_are_todays_rounds(emu, seed, share):
    s = synth(seed, SEEDS[seed])
    budget = scaled_budget(emu, s, share)[0] if share < 1.0 else int(max(min_budget(emu, s, kc) for kc in by_contig(s) if kc) * share)
    unfit, rounds = todays_rounds(emu, s, budget)
    st, units, info = plan(emu, s, budget, False)
    if unfit >= 0:
        assert st == GENERIC_ERROR and info["unfit_contig"] == unfit and share < 1.0
        return
    assert st == SUCCESS and info["split_contigs"] == info["repeat_overlaps"] == 0
    assert [(a, b, ov) for _, a, b, ov, _ in units] == rounds
    assert (len(rounds) == 1) == (share == 4.0)


@pytest.mark.parametrize("case", ["fastq_500", "fasta_500"])
@pytest.mark.parametrize("share", [0.5, 0.25])
def test_lambda_units(emu, case, share):
    s = lambda_columns(case)
    budget, whole = scaled_budget(emu, s, share)
    st, units, info = plan(emu, s, budget, True)
    assert st == SUCCESS
    check_units(s, units)
    assert len(units) >= 1 / share and info["split_contigs"] == 1 and info["repeat_overlaps"] > 0
    st, units1, _ = plan(emu, s, whole, True)
    assert st == SUCCESS and len(units1) == 1 and units1[0][3] == list(range(len(s["t_id"])))


def edge_set(w=W):
    """One contig of 12 windows and a short last one (12 * w + 137 bases), a second of 4: overlaps of two windows each,
    starting or ending exactly on window boundaries, none meeting windows 5 and 6 of the first contig, and one overlap
    over the first contig's whole length."""
    L = 12 * w + 137
    rows = []
    for x in range(12):
        if x in (4, 5, 6):
            continue
        for j in range(6):
            tb = x * w if j % 2 == 0 else x * w + 37 * j
            te = min(L, (x + 2) * w if j % 3 == 0 else tb + w + 11 * j)
            if x in (3,):
                te = min(te, 5 * w)  # window 5 and 6 stay without layers: stop exactly at 5 * w
            rows.append((0, tb, te, te - tb + j, j))
    rows.append((0, 12 * w, L, L - 12 * w, 0))  # the short last window's own overlap
    rows.append((0, 0, L, L, 0))  # the whole contig
    for j in range(10):
        rows.append((2, j * 130, j * 130 + 700, 700, 1))
    rng = np.random.default_rng(5)
    rows = [rows[i] for i in rng.permutation(len(rows))]
    return columns([0, L, L + 300, L + 300 + 4 * w], rows)


def test_edges(emu):
    """every budget from what the fullest window needs to what the whole first contig needs: the units own each window
    once with exactly its overlaps, whatever their boundaries; and over these budgets each edge is reached"""
    s = edge_set()
    ks = by_contig(s)
    lo, hi = spans(s)
    fw = first_windows(s)
    assert ((s["t_end"] % W == 0) & (s["t_end"] > s["t_begin"])).any() and (s["t_begin"] % W == 0).any()
    whole = int(np.flatnonzero((s["t_id"] == 0) & (s["t_begin"] == 0) & (s["t_end"] == s["t_off"][1]))[0])
    # only the whole-contig overlap meets windows 5 and 6: they get no layer from any other
    empty = [x for x in range(13) if all(k == whole for k in ks[0] if lo[k] <= x <= hi[k])]
    assert empty == [5, 6]
    need = max(min_budget(emu, s, [k for k in ks[0] if lo[k] <= x <= hi[k]]) for x in range(13))
    reached = {"three_units": False, "next_to_empty": False, "short_last": False}
    counts = set()
    for budget in np.linspace(need, min_budget(emu, s, ks[0]), 40).astype(np.int64):
        st, units, info = plan(emu, s, int(budget), True)
        assert st == SUCCESS, (budget, info)
        owner = check_units(s, units)
        counts.add(len(units))
        split = [u for u in units if u[4]]
        assert units[-1][0] == 2 and not units[-1][4]  # the small contig is one whole unit
        if not split:
            continue
        assert {u[0] for u in split} == {0} and info["split_contigs"] == 1
        reached["three_units"] |= sum(whole in u[3] for u in units) >= 3
        bounds = {u[1] for u in split[1:]}
        reached["next_to_empty"] |= any(x in bounds or x + 1 in bounds for x in empty)
        last = units[owner[12]]  # the short last window (137 bases) with its own overlap
        reached["short_last"] |= last[1] < 12 and last[2] == 13
    assert all(reached.values()), reached
    assert len(counts) >= 4


def test_window_over_the_budget_is_reported(emu):
    s = edge_set()
    ks = by_contig(s)
    lo, hi = spans(s)
    need = [min_budget(emu, s, [k for k in ks[0] if lo[k] <= x <= hi[k]]) for x in range(13)]
    st, _, info = plan(emu, s, max(need) - 1, True)
    assert st == GENERIC_ERROR and info["unfit_contig"] == 0
    st, _, info = plan(emu, s, max(need), True)
    assert st == SUCCESS and info["unfit_contig"] == -1
    # without splitting, the first contig that does not fit alone
    st, _, info = plan(emu, s, max(need), False)
    assert st == GENERIC_ERROR and info["unfit_contig"] == 0


def test_pair_that_never_fits_is_reported(emu):
    s = columns([0, 3000, 6000], [(1, 0, 800, 800, 0), (0, 100, 900, 900, 0), (1, 600, 2900, 1 << 30, 0)])
    st, _, info = plan(emu, s, 1 << 40, True)
    assert st == GENERIC_ERROR and info["unfit_contig"] == 1


def test_invalid_columns(emu):
    s = columns([0, 3000], [(0, 100, 3001, 900, 0)])  # past the contig's end
    assert plan(emu, s, 1 << 40, True)[0] == INVALID_ARGUMENT
    s = columns([0, 3000], [(1, 100, 900, 900, 0)])  # no such contig
    assert plan(emu, s, 1 << 40, True)[0] == INVALID_ARGUMENT
