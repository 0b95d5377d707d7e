"""GPU (-m gpu): the CUDA DP fill (poa_fill.cuh) cell for cell against its scalar twin, at the edges of every fill
variant and of the shared-memory geometry the host picks for it (fill_cases.py describes the window sets).

On the digest build (racon_gpu_b200/variants/libb200poa_digest.so) every read's fills are hashed; the per-read digests
and fill counts, status, consensus, coverage and MSA rows must equal the emulation's, run at the ring size the launch
reports.  In full band the outputs must also equal the oracle's.  The product library repeats the ladder, ring,
band-256, letter and scoring cases at output level."""
import numpy as np
import pytest

import fill_cases as fc
from emu_lib import Emu

pytestmark = pytest.mark.gpu
CASES = fc.cases()
DIGEST_CASES = list(CASES)
PRODUCT_CASES = ["ladder", "ring", "bands", "letters", "scoring"]


@pytest.fixture(scope="module")
def emu():
    return Emu()


def _check(emu, oracle, runs, results, digest):
    bad = []
    for r, got in zip(runs, results):
        rr = got.get("ring_rows", fc.ring_rows_of(r))
        assert rr == fc.ring_rows_of(r), (r["name"], rr)
        want = fc.emu_run(emu, r, rr)
        assert fc.reach_failures(r["name"], want["reach"], r["batch"], r) == [], r["name"]
        orc = fc.oracle_outputs(oracle, r) if r["mode"] == "full" else None
        bad += fc.compare(r, got, want, orc)
        if not digest:
            assert "digest" not in got
    return bad


@pytest.mark.parametrize("case", DIGEST_CASES)
def test_fill_digests_equal_the_emulation(emu, oracle, case):
    runs = CASES[case]
    results = fc.gpu_runs(runs, digest=True)
    bad = _check(emu, oracle, runs, results, True)
    assert bad == [], "\n".join(bad[:20])
    if case == "ring":  # the consensus does not depend on the ring
        n = runs[0]["batch"].n_windows
        assert results[1]["cons"][:n] == results[0]["cons"]
    if case == "slot_reuse":  # poisoned, reused slots give what clean ones give
        for k in range(0, len(runs), 3):
            for j in (1, 2):
                assert (results[k + j]["digest"] == results[k]["digest"]).all()
                assert results[k + j]["cons"] == results[k]["cons"] and results[k + j]["msa"] == results[k]["msa"]


@pytest.mark.parametrize("case", PRODUCT_CASES)
def test_product_library_outputs_equal_the_emulation(emu, oracle, case):
    runs = CASES[case]
    if case == "bands":
        runs = [r for r in runs if r["band"] == 256]
    results = fc.gpu_runs(runs, digest=False)
    bad = _check(emu, oracle, runs, results, False)
    assert bad == [], "\n".join(bad[:20])
