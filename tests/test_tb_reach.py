"""CPU: every window set of tests/test_gpu_traceback.py reaches the traceback paths its name promises (the emulation's
traceback report), the traceback of every fill equals its scalar twin walk, and in full band every alignment added to
a graph equals spoa's (tb_cases.py describes the cases)."""
import numpy as np
import pytest

import fill_cases as fc
import tb_cases as tc
from emu_lib import Emu

CASES = tc.cases()
RUNS = [(c, i) for c, runs in CASES.items() for i in range(len(runs))]


@pytest.fixture(scope="module")
def emu():
    return Emu()


@pytest.mark.parametrize("case,i", RUNS, ids=[CASES[c][i]["name"] for c, i in RUNS])
def test_case_reaches_its_traceback_paths(emu, oracle, case, i):
    r = CASES[case][i]
    out = fc.emu_run(emu, r, fc.ring_rows_of(r), msa=False)
    assert (out["status"] == 0).all(), out["status"]
    assert tc.mismatch_report(r, out) == []
    assert tc.tb_reach_failures(case, r, out) == []
    b = r["batch"]
    reads = np.setdiff1d(np.arange(b.n_seqs), b.win_seq_off[:-1])
    assert (out["aln_count"][reads] > 0).all()
    if r["mode"] == "full":
        assert fc.aln_digest_failures(r["name"], b, out, tc.oracle_aln(oracle, r), "oracle") == []


def test_aln_digest_depends_on_every_entry(emu, oracle):
    """A change of scoring moves the alignments, and the oracle's digest follows it; a window whose reads equal the
    backbone has one diagonal alignment per read, all with the same digest."""
    r = fc.run("d", fc.synth_windows(4, 300, 8, 0.12, seed=29))
    a = fc.emu_run(emu, r, 8, msa=False)
    c = fc.emu_run(emu, dict(r, scoring=(1, -1, -1)), 8, msa=False)
    reads = a["aln_count"] > 0
    assert (a["aln_digest"][reads] != c["aln_digest"][reads]).any()
    assert fc.aln_digest_failures("d", r["batch"], c, tc.oracle_aln(oracle, dict(r, scoring=(1, -1, -1)))) == []
    truth = fc.ACGT[np.random.default_rng(2).integers(0, 4, 100)].tobytes()
    same = fc.run("same", fc.WindowBatch.from_lists([fc._window([truth] * 4, [None] * 4)]))
    s = fc.emu_run(emu, same, 8, msa=False)
    assert (s["aln_count"][1:] == 100).all() and len(set(s["aln_digest"][1:].tolist())) == 1
