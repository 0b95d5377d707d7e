"""GPU (-m gpu): the CUDA graph phases (poa_core.cuh add_alignment, topsort_roots, mark_subgraph, generate_consensus)
read for read against the emulation and spoa (graph_cases.py describes the window sets).

On the digest build (racon_gpu_b200/variants/libb200poa_digest.so) the graph after every read, the subgraph of every
partial-span read and the consensus scores before and after branch completion are hashed; they, the node and edge
counts, the rounds of branch completion, status, consensus, coverage and MSA rows must equal the emulation's, run at
the ring size the launch reports (the emulation's sort, subgraph and consensus scores are themselves checked against
serial twins).  In full band they must also equal spoa's.  The product library repeats the ties, branch, subgraph and
limits cases at output level; for the limits it also checks what the polisher returns for such windows."""
import numpy as np
import pytest

import fill_cases as fc
import graph_cases as gc
from emu_lib import Emu

pytestmark = pytest.mark.gpu
CASES = gc.cases()
PRODUCT_CASES = ["ties", "branch", "subgraph", "limits"]


@pytest.fixture(scope="module")
def emu():
    return Emu()


def _check(emu, oracle, case, runs, results):
    bad = []
    for r, got in zip(runs, results):
        rr = got.get("ring_rows", fc.ring_rows_of(r))
        assert rr == fc.ring_rows_of(r), (r["name"], rr)
        want = fc.emu_run(emu, r, rr)
        assert gc.mismatch_report(r, want) == [], r["name"]
        assert gc.reach_failures(case, r, want) == [], r["name"]
        ok = np.flatnonzero(want["status"] == 0)
        full = r["mode"] == "full"
        if full and len(ok) < r["batch"].n_windows:  # spoa has no limits: compare the windows the engine finished
            sub = fc.WindowBatch.from_lists([list(zip(*r["batch"].window(int(w)))) for w in ok])
            rs = dict(r, batch=sub)
            orc = fc.oracle_outputs(oracle, rs)
            gs = {k: [got[k][int(w)] for w in ok] for k in ("cons", "cov", "msa", "msa_status")}
            ws = {k: [want[k][int(w)] for w in ok] for k in ("cons", "cov", "msa")}
            ws["status"] = want["status"][ok]
            gs["status"] = got["status"][ok]
            bad += fc.compare(rs, gs, ws, orc)
            bad += fc.compare(dict(r, name=r["name"] + " (all windows)"), got, want)
        else:
            bad += fc.compare(r, got, want, fc.oracle_outputs(oracle, r) if full else None)
        if "graph" in got and full:  # fc.compare has compared the digests with the emulation's
            orc = gc.oracle_graph(oracle, r)
            assert (orc["overflow"] == 0).all(), (r["name"], orc["overflow"])
            bad += fc.graph_digest_failures(r["name"], r["batch"], got["graph"], orc, "oracle", windows=ok)
    return bad


@pytest.mark.parametrize("case", list(CASES))
def test_graphs_equal_the_emulation_and_spoa(emu, oracle, case):
    runs = CASES[case]
    results = fc.gpu_runs(runs, digest=True)
    assert all("graph" in g for g in results)
    bad = _check(emu, oracle, case, runs, results)
    assert bad == [], "\n".join(bad[:20])


@pytest.mark.parametrize("case", PRODUCT_CASES)
def test_product_library_outputs_equal_the_emulation(emu, oracle, case):
    runs = CASES[case]
    results = fc.gpu_runs(runs, digest=False)
    assert all("graph" not in g for g in results)
    bad = _check(emu, oracle, case, runs, results)
    assert bad == [], "\n".join(bad[:20])


def test_windows_the_graph_limits_stop_come_back_as_backbone():
    """A window that stops on a graph limit (a ninth letter in one column, one node past max_nodes, an in-degree of
    256) reports its status and the polisher returns its backbone, never a hole; the window next to it is polished."""
    from racon_gpu_b200 import api
    for r in CASES["limits"]:
        b = r["batch"]
        pol = api.Polisher(devices=[0], mem_per_batch=fc.GB, max_sequence_size=r["msz"],
                           max_sequences_per_poa=r["depth"])
        cons, clen, polished, status = pol.polish(b, tgs=True, trim=True)
        pol.close()
        got = api.consensus_list(cons, clen)
        for w, want in enumerate(gc.LIMIT_STATUS[r["name"]]):
            assert int(status[w]) == want, (r["name"], w, status.tolist())
            if want:
                assert not polished[w] and got[w] == b.window(w)[0][0], (r["name"], w)
            else:
                assert polished[w] and len(got[w]) > 0, (r["name"], w)
