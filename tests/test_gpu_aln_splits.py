"""GPU (-m gpu): every Hirschberg split of the overlap aligner against the emulation, on one warp and on warp teams
(aln_cases.py describes the batches).

On the digest build (racon_gpu_b200/variants/libb200poa_digest.so) the split kernels log every split attempt with
hashes of both middle columns.  The device's log must equal the emulation's records as a set keyed by (alignment, r0,
c0, n, m, attempt): band, level, split and hashes.  No team_wait may have given up, every case must show the paths it
names (one warp, a thin level's team, the side stream's team), and every CIGAR must be the oracle's.  The product
library repeats a subset at output level."""
import os

import numpy as np
import pytest

import aln_cases as ac
from emu_lib import EmuAligner
from oracle_lib import ops_to_cigar, oracle_align
from racon_gpu_b200.aligner import SPLIT_PATHS, SPLIT_TIMEOUT

pytestmark = pytest.mark.gpu
CASES = ac.cases()
PRODUCT_CASES = ["stripe_edges", "guesses", "saturated", "cursor"]


@pytest.fixture(scope="module")
def emu():
    return EmuAligner()


_ORACLE = {}


def _oracle_cigars(oracle, pairs):
    """(edit distance, CIGAR) of every pair, computed once (ctypes calls run outside the GIL: a thread each)."""
    from concurrent.futures import ThreadPoolExecutor

    def one(pair):
        ops, score = oracle_align(oracle, *pair)
        return score, ops_to_cigar(oracle, ops)

    todo = [p for p in dict.fromkeys(pairs) if p not in _ORACLE]
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        for p, v in zip(todo, ex.map(one, todo)):
            _ORACLE[p] = v
    return [_ORACLE[p] for p in pairs]


def _cigar_failures(oracle, r, res):
    bad = []
    want = _oracle_cigars(oracle, r["pairs"])
    for rnd, got in enumerate(res["rounds"]):
        for k, (q, t) in enumerate(r["pairs"]):
            score, cigar = want[k]
            if got["ed"][k] != score or got["cigars"][k] != cigar:
                bad.append(f"{r['name']} round {rnd}: alignment {k} ({len(q)}x{len(t)}) differs from the oracle")
    return bad


@pytest.mark.parametrize("case", list(CASES))
def test_split_log_equals_the_emulation(emu, oracle, case):
    runs = CASES[case]
    results = ac.gpu_runs(runs, digest=True)
    bad = []
    for r, res in zip(runs, results):
        want = ac.emu_records(emu, r)
        for rnd, (log, (recs, _)) in enumerate(zip(res["logs"], want)):
            bad += ac.compare_logs(f"{r['name']} round {rnd}", log, recs)
            timed_out = log[(log["flags"] & SPLIT_TIMEOUT) != 0]
            if timed_out.shape[0]:
                x = timed_out[0]
                bad.append(f"{r['name']}: a team_wait gave up in alignment {int(x['aln'])} sub-problem {int(x['n'])}x{int(x['m'])}")
        paths = {SPLIT_PATHS[int(p)] for log in res["logs"] for p in log["path"]}
        info = res["rounds"][0]["info"]
        for p in r["paths"]:
            if p not in paths:
                bad.append(f"{r['name']}: no split took the path {p} (paths {sorted(paths)}, {info['n_team_blocks']} team blocks)")
        if r["no_teams"] and (info["n_team_blocks"] != 0 or paths != {"warp"}):
            bad.append(f"{r['name']}: {info['n_team_blocks']} team blocks, paths {sorted(paths)}")
        if r["more_items_than_blocks"]:
            lv = [x["level"] for x in res["logs"][0] if x["path"] == 1 and x["attempt"] == 0]
            if not lv or np.bincount(lv).max() <= info["n_team_blocks"]:
                bad.append(f"{r['name']}: no level had more team work items than its {info['n_team_blocks']} team blocks")
        bad += _cigar_failures(oracle, r, res)
    if case == "guesses" or case == "saturated":  # the redo on every path
        redo = {SPLIT_PATHS[int(x["path"])] for res in results for log in res["logs"] for x in log if x["attempt"] == 1}
        need = {"warp", "team"} if case == "guesses" else {"warp", "side", "team"}
        if not need <= redo:
            bad.append(f"{case}: redone splits on {sorted(redo)}, expected {sorted(need)}")
    if case == "cursor":  # the same pairs on teams and on one warp: the same records, hash for hash
        for rnd in range(2):
            a, b = results[0]["logs"][rnd], results[1]["logs"][rnd]
            bad += ac.compare_logs(f"cursor round {rnd}: one warp against teams", b, a)
    assert bad == [], "\n".join(bad[:20])


@pytest.mark.parametrize("case", PRODUCT_CASES)
def test_product_library_cigars_equal_the_oracle(oracle, case):
    runs = CASES[case]
    results = ac.gpu_runs(runs, digest=False)
    bad = []
    for r, res in zip(runs, results):
        assert res["logs"] == []
        bad += _cigar_failures(oracle, r, res)
    assert bad == [], "\n".join(bad[:20])
