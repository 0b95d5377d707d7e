"""CPU: every Hirschberg split of the overlap aligner's cases (aln_cases.py), column for column.

The emulation (tests/emu, aln_core.cuh in its host flavour) runs each split sub-problem the way the split kernels do:
on one warp, and on a team block of 2 x ALN_TEAM threads whose hand-over protocol is checked word by word (shadow
tags of the writer's pass and stripe, and the wait contract).  Both middle columns must equal each other and obey the
band contract of myers_pass against the plain distance matrix (oracle/aln_oracle.c): with band b every value <= b - 2
is exact, every other one is an overestimate, ALN_INF only in rows whose strip ends before the last column; and the
split must be the one the split rule gives on the exact columns whenever the optimum is <= b - 2."""
import functools

import numpy as np
import pytest

import aln_cases as ac
from emu_lib import EmuAligner
from oracle_lib import Oracle, oracle_last_column

INF = 1 << 28
TEAM_RUNS = ["stripe_edges_whole", "stripe_edges_banded", "word_edges", "tiny_bands", "tall_thin", "guesses", "letters",
             "letters_banded", "huge_thin", "cursor"]


@pytest.fixture(scope="module")
def emu():
    return EmuAligner()


@pytest.fixture(scope="module")
def orc():
    return Oracle()


def _runs():
    return {r["name"]: r for runs in ac.cases().values() for r in runs}


@functools.lru_cache(maxsize=None)
def _subproblems(name):
    """Every split attempt the run's first round makes (one-warp emulation's records): (record, q, t) of each."""
    r = _runs()[name]
    recs = ac.emu_records(EmuAligner(), dict(r, rounds=1))[0][0]
    out = []
    for x in recs:
        q, t = r["pairs"][int(x["aln"])]
        out.append((x, q[x["r0"]:x["r0"] + x["n"]], t[x["c0"]:x["c0"] + x["m"]]))
    return out


def exact_columns(orc, q, t):
    lh = len(t) // 2
    return oracle_last_column(orc, q, t[:lh]), oracle_last_column(orc, q[::-1], t[lh:][::-1])


def split_rule(L, R, m):
    """edlib.cpp:1282-1308 on two columns: (r, ls, rs, best)"""
    n = L.shape[0] - 1
    lh, rh = m // 2, m - m // 2
    sums = L[1:n] + R[n - 1:0:-1] if n >= 2 else np.zeros(0, dtype=np.int64)
    top, bot = lh + int(R[n]), int(L[n]) + rh
    best = min([top, bot] + ([int(sums.min())] if sums.shape[0] else []))
    hit = np.flatnonzero(sums == best)
    if hit.shape[0]:
        r = int(hit[0])
        return r, int(L[r + 1]), int(R[n - r - 1]), best
    if top == best:
        return -1, lh, best - lh, best
    return n - 1, best - rh, rh, best


def band_failures(where, col, exact, band, n, cols):
    """myers_pass's band contract for one middle column"""
    bad = []
    if band < 0:
        if not (col == exact).all():
            i = int(np.flatnonzero(col != exact)[0])
            bad.append(f"{where}: row {i} = {col[i]}, the matrix has {exact[i]} (no band)")
        return bad
    rows = np.arange(n + 1)
    stripe = np.maximum(rows - 1, 0) // ac.STRIPE
    R0, R1 = ac.STRIPE * stripe, np.minimum(ac.STRIPE * (stripe + 1), n)
    may_be_inf = (R1 + band - 1 < cols - 1) | (R0 - band > cols - 1)
    may_be_inf[0] = False
    need = exact <= band - 2
    for what, mask in (("is not exact", need & (col != exact)), ("underestimates", col < exact),
                       ("is ALN_INF where the strip reaches the last column", (col == INF) & ~may_be_inf)):
        if mask.any():
            i = int(np.flatnonzero(mask)[0])
            bad.append(f"{where}: band {band}, row {i} = {col[i]} {what} (the matrix has {exact[i]})")
    return bad


def check_split(emu, orc, x, q, t, seed=1):
    """All checks of one split sub-problem; returns (failures, team stats)."""
    where = f"alignment {int(x['aln'])} sub-problem r0={int(x['r0'])} c0={int(x['c0'])} {len(q)}x{len(t)} attempt {int(x['attempt'])}"
    band = int(x["band"])
    best = band - 2 if band >= 0 else -1
    warp = emu.split(q, t, best=best)[0]
    team = emu.split(q, t, best=best, team=True, seed=seed)[0]
    stats, failure = emu.last_stats, emu.last_failure
    bad = []
    if stats["failures"] or stats["timeouts"]:
        bad.append(f"{where}: team protocol: {failure} ({stats['failures']} failures, {stats['timeouts']} timeouts)")
    for k in ("Lc", "Rr"):
        if not (team[k] == warp[k]).all():
            i = int(np.flatnonzero(team[k] != warp[k])[0])
            bad.append(f"{where}: team {k}[{i}] = {team[k][i]}, one warp {warp[k][i]}")
    if [team[k] for k in ("r", "ls", "rs", "best")] != [warp[k] for k in ("r", "ls", "rs", "best")]:
        bad.append(f"{where}: team split {[team[k] for k in ('r', 'ls', 'rs', 'best')]} != one warp's")
    if [warp[k] for k in ("r", "ls", "rs", "best")] != [int(x[k]) for k in ("r", "ls", "rs", "best")]:
        bad.append(f"{where}: the split differs from the batch emulation's record")
    L, R = exact_columns(orc, q, t)
    lh = len(t) // 2
    bad += band_failures(where + " Lc", warp["Lc"], L, band, len(q), lh)
    bad += band_failures(where + " Rr", warp["Rr"], R, band, len(q), len(t) - lh)
    want = split_rule(L, R, len(t))
    if band < 0 or want[3] <= band - 2:
        got = tuple(warp[k] for k in ("r", "ls", "rs", "best"))
        if got != want:
            bad.append(f"{where}: split {got}, the exact columns give {want}")
    return bad, stats


@pytest.mark.parametrize("name", TEAM_RUNS)
def test_every_split_equals_the_plain_matrix_on_one_warp_and_on_a_team(emu, orc, name):
    """Every split attempt of the run (every level, the redone ones too): team == one warp, protocol clean, band
    contract against the plain matrix, split rule on the exact columns.  Then the case reaches what its name promises."""
    subs = _subproblems(name)
    bad = []
    reach = {k: 0 for k in EmuAligner.SPLIT_STATS}
    max_stripes, bands, odd_even, redo_shapes = 0, set(), set(), set()
    for x, q, t in subs:
        b, stats = check_split(emu, orc, x, q, t)
        bad += b
        for k in reach:
            reach[k] += stats[k]
        max_stripes = max(max_stripes, (len(q) + ac.STRIPE - 1) // ac.STRIPE)
        if len(q) > ac.STRIPE:
            odd_even.add(len(t) % 2)
            if x["level"] == 0 and x["band"] >= 0:
                bands.add(int(x["band"]) % 16)
        if x["attempt"] == 1:
            redo_shapes.add("team" if len(q) > ac.STRIPE else "warp")
    assert bad == [], "\n".join(bad[:20])
    # what the name promises
    if name.startswith("stripe_edges"):
        assert max_stripes > 4 and odd_even == {0, 1}, (max_stripes, odd_even)  # the ring wraps; lh == rh and lh != rh
        ns = {len(q) for x, q, t in subs if x["level"] == 0}
        assert all(ac.STRIPE * k + d in ns for k in range(1, 7) for d in (-64, -1, 0, 1, 63, 64))
    if name == "word_edges":
        assert {0, 1, 15} <= bands, bands
    if name == "tiny_bands":
        assert reach["anchors"] > 0
    if name == "tall_thin":
        assert reach["left_matrix"] > 0
    if name == "guesses":
        assert redo_shapes == {"warp", "team"}, redo_shapes
    if name.startswith("letters"):
        assert reach["other"] > 0
    if name == "huge_thin":
        assert any(x["n"] >= 8192 and int(x["n"]) * int(x["m"]) >= 32 << 20 for x, q, t in subs)
        assert redo_shapes == {"team"}
    assert reach["waits"] > 0


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4, 5])
def test_team_protocol_holds_under_several_schedules(emu, seed):
    """The team pipeline's largest, banded, anchored, redone and non-ACGT sub-problems under different random yields."""
    picks = []
    for name in ("stripe_edges_banded", "tiny_bands", "tall_thin", "letters_banded", "huge_thin"):
        subs = [s for s in _subproblems(name) if len(s[1]) > ac.STRIPE]
        subs.sort(key=lambda s: -len(s[1]))
        picks += subs[:2]
    for x, q, t in picks:
        band = int(x["band"])
        warp = emu.split(q, t, best=band - 2 if band >= 0 else -1)[0]
        team = emu.split(q, t, best=band - 2 if band >= 0 else -1, team=True, seed=100 + seed)[0]
        st = emu.last_stats
        assert st["failures"] == 0 and st["timeouts"] == 0, emu.last_failure
        assert (team["Lc"] == warp["Lc"]).all() and (team["Rr"] == warp["Rr"]).all(), (int(x["aln"]), len(q), len(t))


def test_the_redo_rule_runs_a_second_pass_in_the_same_team_block(emu, orc):
    """A guess that proves too small: the team block runs the whole sub-problem again (the progress words and hand-over
    rows of the first pass are still there) and the second attempt is exact."""
    r = _runs()["guesses"]
    for q, t in r["pairs"]:
        g = ac.guess_of(len(q), len(t), r["permille"])
        if len(q) <= ac.STRIPE:
            continue
        att = emu.split(q, t, best=g, guess=True, team=True, seed=7)
        assert emu.last_stats["failures"] == 0, emu.last_failure
        L, R = exact_columns(orc, q, t)
        if len(att) == 2:
            assert att[0]["best"] > g and att[1]["band"] == -1
            assert (att[1]["Lc"] == L).all() and (att[1]["Rr"] == R).all()
        else:
            assert att[0]["best"] <= g and att[0]["best"] == split_rule(L, R, len(t))[3]
