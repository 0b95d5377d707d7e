"""CPU: every window set of tests/test_gpu_fill.py reaches the DP-fill path its name promises (the emulation's reach
report, at the ring size the GPU launch will use), and in full band the emulation equals the oracle on it."""
import numpy as np
import pytest

import fill_cases as fc
from emu_lib import Emu

CASES = fc.cases()
RUNS = [(c, i) for c, runs in CASES.items() for i in range(len(runs))]


@pytest.fixture(scope="module")
def emu():
    return Emu()


@pytest.mark.parametrize("case,i", RUNS, ids=[CASES[c][i]["name"] for c, i in RUNS])
def test_case_reaches_its_fill_path(emu, oracle, case, i):
    r = CASES[case][i]
    out = fc.emu_run(emu, r, fc.ring_rows_of(r), msa=False)
    assert (out["status"] == 0).all(), out["status"]
    assert fc.reach_failures(r["name"], out["reach"], r["batch"], r) == []
    # every read of every window was filled at least once
    b = r["batch"]
    assert (out["count"][np.setdiff1d(np.arange(b.n_seqs), b.win_seq_off[:-1])] > 0).all()
    if r["mode"] == "full" and not r["env"]:
        oc, ocov, _ = fc.oracle_outputs(oracle, r, msa=False)
        assert out["cons"] == oc
        assert all(np.array_equal(a, c) for a, c in zip(out["cov"], ocov))


def test_digest_depends_on_every_cell_and_not_on_the_ring(emu):
    """The digest sees a change of scoring (every cell moves) and of band width, and a ring size changes only the row
    program's far flags, never the matrix."""
    r = fc.run("d", fc.synth_windows(4, 300, 8, 0.12, seed=29))
    a = fc.emu_run(emu, r, 8, msa=False)
    b = fc.emu_run(emu, r, 2, msa=False)
    assert (a["digest"] == b["digest"]).all() and a["reach"]["far_preds"].sum() < b["reach"]["far_preds"].sum()
    c = fc.emu_run(emu, dict(r, scoring=(3, -5, -5)), 8, msa=False)
    d = fc.emu_run(emu, dict(r, mode="static", band=128), 8, msa=False)
    reads = a["count"] > 0
    assert (a["digest"][reads] != c["digest"][reads]).all() and (a["digest"][reads] != d["digest"][reads]).all()
