"""GPU (-m gpu): every leaf of the overlap aligner against the emulation, and the CIGARs, operations and breaking points
formed from them against the oracle (aln_leaf_cases.py describes the batches).

On the digest build (racon_gpu_b200/variants/libb200poa_digest.so) the leaf kernel logs every leaf with its end score,
a hash of its operations region and the walk's counters.  The device's log must equal the emulation's records as a set
keyed by (alignment, r0, c0, n, m), with no leaf twice, none missing and no overflow, and every CIGAR must be the
oracle's.  The same batch object then aligns the case again after a round of larger, heavily edited pairs, and a fresh
batch aligns it in reverse order: the slots hold other leaves' records then, and the log must not change.  The product
library repeats every case at output level: CIGARs, operations and breaking points, with and without CIGAR text."""
import os

import numpy as np
import pytest

import aln_leaf_cases as lc
from emu_lib import EmuAligner
from oracle_lib import ops_to_cigar, oracle_align, oracle_breaking_points

pytestmark = pytest.mark.gpu
CASES = lc.cases()


@pytest.fixture(scope="module")
def emu():
    return EmuAligner()


_ORACLE = {}


def _oracle(oracle, pairs):
    """(ops, edit distance, CIGAR) of every pair, computed once (ctypes calls run outside the GIL: a thread each)."""
    from concurrent.futures import ThreadPoolExecutor

    def one(pair):
        q, t = pair
        if not q or not t:
            ops = np.full(len(q) + len(t), 2 if not q else 1, dtype=np.uint8)
            return ops, len(q) + len(t), ops_to_cigar(oracle, ops)
        ops, score = oracle_align(oracle, q, t)
        return ops, score, ops_to_cigar(oracle, ops)

    todo = [p for p in dict.fromkeys(pairs) if p not in _ORACLE]
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        for p, v in zip(todo, ex.map(one, todo)):
            _ORACLE[p] = v
    return [_ORACLE[p] for p in pairs]


def _output_failures(oracle, r, res, tag):
    bad = []
    w = r["window_length"]
    for k, ((q, t), (q_first, t_begin), (ops, score, cigar)) in enumerate(zip(r["pairs"], r["coords"], _oracle(oracle, r["pairs"]))):
        where = f"{r['name']} {tag}: alignment {k} ({len(q)}x{len(t)})"
        if "cigars" in res and (res["ed"][k] != score or res["cigars"][k] != cigar):
            bad.append(f"{where}: CIGAR / distance differ from the oracle")
        if res["ops"][k].shape != ops.shape or not (res["ops"][k] == ops).all():
            bad.append(f"{where}: operations differ from the oracle")
        if w:
            want = oracle_breaking_points(oracle, ops, q_first, t_begin, t_begin + len(t), w)
            if res["bp"][k].shape != want.shape or not (res["bp"][k] == want).all():
                bad.append(f"{where}: breaking points differ from the oracle (window length {w})")
    return bad


@pytest.mark.parametrize("case", list(CASES))
def test_leaf_log_equals_the_emulation(emu, oracle, case):
    runs = CASES[case]
    results = lc.gpu_runs(runs, digest=True)
    bad = []
    for r, res in zip(runs, results):
        want, _ = lc.emu_leaves(emu, r)
        for tag in ("plain", "after_noise", "reversed"):
            got = res[tag]
            bad += lc.compare_logs(f"{r['name']} {tag}", got["log"], want)
            if got["log"].shape[0] != want.shape[0] or got["info"]["n_leaves"] != want.shape[0]:
                bad.append(f"{r['name']} {tag}: {got['log'].shape[0]} leaves logged, {got['info']['n_leaves']} run, "
                           f"the emulation has {want.shape[0]}")
            bad += _output_failures(oracle, r, got, tag)
    assert bad == [], "\n".join(bad[:20])


@pytest.mark.parametrize("case", list(CASES))
def test_product_library_outputs_equal_the_oracle(oracle, case):
    runs = CASES[case]
    results = lc.gpu_runs(runs, digest=False)
    bad = []
    for r, res in zip(runs, results):
        assert set(res) == ({False, True} if r["window_length"] else {False})
        for skip, got in res.items():
            assert "log" not in got
            bad += _output_failures(oracle, r, got, "without CIGAR text" if skip else "with CIGAR text")
    assert bad == [], "\n".join(bad[:20])
