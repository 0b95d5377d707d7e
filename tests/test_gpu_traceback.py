"""GPU (-m gpu): the CUDA traceback (poa_core.cuh traceback(), traceback_i32()) read for read against the emulation and
spoa, at the edges of its tile (tb_cases.py describes the window sets).

On the digest build (racon_gpu_b200/variants/libb200poa_digest.so) every alignment added to a graph is hashed; the
per-read alignment digests and entry counts, fill digests, status, consensus, coverage and MSA rows must equal the
emulation's, run at the ring size the launch reports (the emulation's traceback is itself checked against a scalar twin
walk).  In full band the alignments and outputs must also equal the oracle's.  The product library repeats the band-256,
ends and hubs cases at output level."""
import pytest

import fill_cases as fc
import tb_cases as tc
from emu_lib import Emu

pytestmark = pytest.mark.gpu
CASES = tc.cases()
PRODUCT_CASES = ["band_edges", "ends", "hubs"]


@pytest.fixture(scope="module")
def emu():
    return Emu()


def _check(emu, oracle, case, runs, results):
    bad = []
    for r, got in zip(runs, results):
        rr = got.get("ring_rows", fc.ring_rows_of(r))
        assert rr == fc.ring_rows_of(r), (r["name"], rr)
        want = fc.emu_run(emu, r, rr)
        assert tc.mismatch_report(r, want) == [], r["name"]
        assert tc.tb_reach_failures(case, r, want) == [], r["name"]
        orc = fc.oracle_outputs(oracle, r) if r["mode"] == "full" else None
        bad += fc.compare(r, got, want, orc)
        if "aln_digest" in got and r["mode"] == "full":
            bad += fc.aln_digest_failures(r["name"], r["batch"], got, tc.oracle_aln(oracle, r), "oracle")
    return bad


@pytest.mark.parametrize("case", list(CASES))
def test_alignments_equal_the_emulation_and_spoa(emu, oracle, case):
    runs = CASES[case]
    results = fc.gpu_runs(runs, digest=True)
    assert all("aln_digest" in g for g in results)
    bad = _check(emu, oracle, case, runs, results)
    assert bad == [], "\n".join(bad[:20])


@pytest.mark.parametrize("case", PRODUCT_CASES)
def test_product_library_outputs_equal_the_emulation(emu, oracle, case):
    runs = CASES[case]
    if case == "band_edges":
        runs = [r for r in runs if r["band"] == 256]
    results = fc.gpu_runs(runs, digest=False)
    assert all("aln_digest" not in g for g in results)
    bad = _check(emu, oracle, case, runs, results)
    assert bad == [], "\n".join(bad[:20])
