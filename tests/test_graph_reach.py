"""CPU: every window set of tests/test_gpu_graph.py reaches the paths of add_alignment, the sorts, the subgraph and the
consensus its name promises (the emulation's graph report), the per-root sort, the warp-sweep subgraph and the blocked
consensus scores equal their serial twins on every read, and in full band every graph, subgraph and consensus digest
equals spoa's (graph_cases.py describes the cases)."""
import numpy as np
import pytest

import fill_cases as fc
import graph_cases as gc
from emu_lib import Emu

CASES = gc.cases()
RUNS = [(c, i) for c, runs in CASES.items() for i in range(len(runs))]


@pytest.fixture(scope="module")
def emu():
    return Emu()


@pytest.mark.parametrize("case,i", RUNS, ids=[CASES[c][i]["name"] for c, i in RUNS])
def test_case_reaches_its_graph_paths(emu, oracle, case, i):
    r = CASES[case][i]
    out = fc.emu_run(emu, r, fc.ring_rows_of(r), msa=False)
    assert gc.mismatch_report(r, out) == []
    assert gc.reach_failures(case, r, out) == []
    b = r["batch"]
    ok = np.flatnonzero(out["status"] == 0)
    assert (out["graph"]["graph_nodes"][b.win_seq_off[:-1][ok]] > 0).all()
    if r["mode"] == "full":
        orc = gc.oracle_graph(oracle, r)
        assert (orc["overflow"] == 0).all(), orc["overflow"]
        assert fc.graph_digest_failures(r["name"], b, out["graph"], orc, "oracle", windows=ok) == []
        for w in np.flatnonzero(out["status"] != 0):  # a window stopped on a limit: every read it did add, as spoa
            s0, s1 = int(b.win_seq_off[w]), int(b.win_seq_off[w + 1])
            done = [s for s in range(s0, s1) if out["graph"]["graph_nodes"][s] > 0]
            assert done, (r["name"], int(w))
            for f in ("graph_digest", "graph_nodes", "graph_edges", "sub_digest", "sub_count"):
                assert (out["graph"][f][done] == orc[f][done]).all(), (r["name"], int(w), f)
        if r["name"] == "limits_indegree":  # the hub really holds 255 and 256 in-edges
            assert orc["max_indegree"].tolist() == gc.HUB_INDEGREE


def test_graph_digest_depends_on_every_field(emu):
    """A weight, a letter or an edge more changes the digest: reads equal to the backbone give the same graph digest
    at every read except for the weights (which grow), and the same window with per-base weights differs."""
    truth = fc.ACGT[np.random.default_rng(3).integers(0, 4, 80)].tobytes()
    same = fc.run("same", fc.WindowBatch.from_lists([fc._window([truth] * 4, [None] * 4)]))
    a = fc.emu_run(emu, same, 8, msa=False)["graph"]
    assert (a["graph_nodes"] == 80).all() and (a["graph_edges"] == 79).all()
    assert len(set(a["graph_digest"].tolist())) == 4
    wts = [np.full(80, 5, dtype=np.int8)] * 4
    heavy = fc.run("heavy", fc.WindowBatch.from_lists([fc._window([truth] * 4, wts)]))
    c = fc.emu_run(emu, heavy, 8, msa=False)["graph"]
    assert (c["graph_digest"] != a["graph_digest"]).all()
    assert (c["cons_digest"] != a["cons_digest"]).all()
