"""GPU: polishing from aligned overlaps with several workers (b200poa_polish_overlaps_multi, api.polish_overlaps with
devices=) against the single-device call window for window -- consensus, polished, status and the export byte for byte
-- on one H100 with repeated device ids for several workers; a contig too large for one aligner batch split at window
boundaries; the lambda sample in several units against racon; and the errors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from common import contig_edit_distance, lambda_fixture, lambda_reference
from overlap_cases import polish_args, synth_overlap_set
from test_gpu_overlap_polish import SETS, THR, W, SCORES
from test_layer_cut import lambda_overlaps

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
WORKERS = ([0], [0, 0], [0, 0, 0], [])


def _same_export(a, b):
    (ia, ba), (ib, bb) = a, b
    assert ia.tobytes() == ib.tobytes()
    for f in ("win_seq_off", "seq_off", "bases", "weights", "has_weights", "begins", "ends"):
        assert getattr(ba, f).tobytes() == getattr(bb, f).tobytes(), f


def _same(want, got):
    assert got[0] == want[0]
    assert (got[1] == want[1]).all() and (got[2] == want[2]).all()
    if "export" in want[3]:
        _same_export(want[3]["export"], got[3]["export"])
    for k in ("tier2_windows", "tier2_polished", "exported_windows", "exported_bytes"):
        if k in want[3]:
            assert got[3][k] == want[3][k], k


@pytest.mark.parametrize("seed", list(SETS))
@pytest.mark.parametrize("with_t_qual", [True, False])
@pytest.mark.parametrize("deep,export", [(False, False), (True, True), (False, True)])
def test_workers_equal_the_single_device_call(seed, with_t_qual, deep, export):
    from racon_gpu_b200 import api
    s = synth_overlap_set(seed, **SETS[seed])
    kw = dict(window_length=W, quality_threshold=THR, mem_per_poa_batch=1 << 30, poa_batches=2, max_windows_per_batch=3,
              deep_windows=deep, export_layers=export, **SCORES)
    want = api.polish_overlaps(**polish_args(s, with_t_qual), **kw)
    if SETS[seed] and export:  # the deep set reaches the second tier, or without it the export
        assert want[3]["tier2_windows"] > 0 if deep else want[3]["exported_windows"] > 0
    for devices in WORKERS:
        got = api.polish_overlaps(**polish_args(s, with_t_qual), devices=devices, **kw)
        _same(want, got)
        assert got[3]["rounds"] == want[3]["rounds"] and got[3]["split_contigs"] == got[3]["repeat_overlaps"] == 0
    # small aligner batches: more units than rounds of whole contigs, same outputs
    if not SETS[seed]:
        got = api.polish_overlaps(**polish_args(s, with_t_qual), devices=[0, 0], **{**kw, "aligner_mem": 4 << 20})
        _same(want, got)
        assert got[3]["rounds"] >= 2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_units") / "libunits_emu.so"
    subprocess.run(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-o", str(so), "-x", "c++",
                    os.path.join(HERE, "emu", "emu_units.cpp")], check=True)
    return C.CDLL(str(so))


def _planner_columns(s):
    import test_overlap_units as tu
    return tu.columns(s["t_off"], [(int(s["t_id"][k]), int(s["t_begin"][k]), int(s["t_end"][k]),
                                    int(s["q_off"][k + 1] - s["q_off"][k]), int(s["q_first"][k]))
                                   for k in range(len(s["t_id"]))])


def _seed13():
    return synth_overlap_set(13, contig_lengths=(500, 30000), depth=40, read_len=(300, 500))


@pytest.mark.parametrize("devices", [[0], [0, 0]])
def test_contig_too_large_for_one_aligner_batch_is_split(devices):
    from racon_gpu_b200 import api
    s = _seed13()
    kw = dict(window_length=W, quality_threshold=THR, mem_per_poa_batch=1 << 30, export_layers=True, **SCORES)
    want = api.polish_overlaps(**polish_args(s), **kw)
    assert want[3]["rounds"] == 1
    got = api.polish_overlaps(**polish_args(s), devices=devices, aligner_mem=4 << 20, **kw)
    _same(want, got)
    info = got[3]
    assert info["split_contigs"] == 1 and info["repeat_overlaps"] > 0 and info["rounds"] >= 3, info
    assert sum(want[1]) > len(want[1]) // 2


@pytest.mark.parametrize("case,golden", [("fastq_500", 1312), ("fasta_500", 1566)])
def test_lambda_in_several_units_like_racon(oracle, case, golden):
    from racon_gpu_b200 import api
    b, cons, polished, p = lambda_fixture(case)
    ov = lambda_overlaps(case)
    contig = b"".join(b.bases[b.seq_off[s]:b.seq_off[s + 1]].tobytes() for s in b.win_seq_off[:-1])
    q = np.frombuffer(b"".join(o["q"] for o in ov), np.uint8).copy()
    q_off = np.concatenate([[0], np.cumsum([len(o["q"]) for o in ov])]).astype(np.int64)
    qual = np.frombuffer(b"".join(o["qual"] if o["qual"] is not None else b"!" * len(o["q"]) for o in ov), np.uint8)
    for devices in ([0], [0, 0, 0]):
        got, gp, gs, info = api.polish_overlaps(
            np.frombuffer(contig, np.uint8), np.asarray([0, len(contig)]), None, np.zeros(len(ov), np.int32),
            np.asarray([o["t_begin"] for o in ov]), np.asarray([o["t_begin"] + len(o["t"]) for o in ov]), q, q_off, qual,
            np.asarray([o["qual"] is not None for o in ov], np.uint8), np.asarray([o["q_first"] for o in ov]),
            window_length=p["window_length"], quality_threshold=10.0, match=p["m"], mismatch=p["x"], gap=p["g"],
            tgs=p["tgs"], trim=p["trim"], mem_per_poa_batch=2 << 30, aligner_mem=12 << 20, devices=devices)
        assert info["rounds"] >= 3 and info["split_contigs"] == 1 and info["repeat_overlaps"] > 0, info
        assert (gp == polished).all() and got == cons
        assert contig_edit_distance(oracle, got, lambda_reference()) == golden


def test_budget_under_one_window_names_the_contig(emu):
    """the smallest budget for contig 0 whole (from the planner's host build) is too small for one window of contig 1"""
    from racon_gpu_b200 import api
    import test_overlap_units as tu
    lib = emu
    s = _seed13()
    cols = _planner_columns(s)
    ks = tu.by_contig(cols)
    budget = tu.min_budget(lib, cols, ks[0])
    assert tu.plan(lib, cols, budget, True)[2]["unfit_contig"] == 1
    with pytest.raises(RuntimeError, match="contig 1 do not fit"):
        api.polish_overlaps(**polish_args(s), window_length=W, quality_threshold=THR, aligner_mem=budget,
                            mem_per_poa_batch=1 << 30, devices=[0, 0], **SCORES)
    # the call returned: the device still polishes
    got = api.polish_overlaps(**polish_args(s), window_length=W, quality_threshold=THR, aligner_mem=4 << 20,
                              mem_per_poa_batch=1 << 30, devices=[0], **SCORES)
    assert got[3]["split_contigs"] == 1


def test_invalid_device_id():
    from racon_gpu_b200 import api
    import torch
    s = synth_overlap_set(11)
    for devices in ([torch.cuda.device_count()], [0, -1]):
        with pytest.raises(RuntimeError, match="invalid_argument"):
            api.polish_overlaps(**polish_args(s), window_length=W, quality_threshold=THR, mem_per_poa_batch=1 << 30,
                                devices=devices, **SCORES)


def test_default_memory_shares_give_the_same_outputs():
    """mem_per_poa_batch and aligner_mem 0: each worker's share shrinks with the workers on the device"""
    from racon_gpu_b200 import api
    s = synth_overlap_set(14, **SETS[14])
    kw = dict(window_length=W, quality_threshold=THR, deep_windows=True, export_layers=True, **SCORES)
    want = api.polish_overlaps(**polish_args(s), **kw)
    for devices in ([0], [0, 0], [0, 0, 0]):
        _same(want, api.polish_overlaps(**polish_args(s), devices=devices, **kw))


def _join(a, b):
    """contigs of b after those of a"""
    nb = a["t_bases"].shape[0]
    return dict(t_bases=np.concatenate([a["t_bases"], b["t_bases"]]), t_off=np.concatenate([a["t_off"], b["t_off"][1:] + nb]),
                t_qual=np.concatenate([a["t_qual"], b["t_qual"]]),
                t_id=np.concatenate([a["t_id"], b["t_id"] + len(a["t_off"]) - 1]).astype(np.int32),
                t_begin=np.concatenate([a["t_begin"], b["t_begin"]]), t_end=np.concatenate([a["t_end"], b["t_end"]]),
                q_bases=np.concatenate([a["q_bases"], b["q_bases"]]),
                q_off=np.concatenate([a["q_off"], b["q_off"][1:] + a["q_off"][-1]]),
                q_qual=np.concatenate([a["q_qual"], b["q_qual"]]),
                has_quality=np.concatenate([a["has_quality"], b["has_quality"]]),
                q_first=np.concatenate([a["q_first"], b["q_first"]]))


def test_second_tier_outcome_does_not_depend_on_the_worker_or_the_split(emu):
    """Contig 0 is the deep set with 1100-base insertions: a worker that polishes it keeps a second-tier batch larger
    than 1023 bases.  Contig 1 has windows of about 600 layers in which a dozen reads carry 1100 random bases each, so
    that their graphs spread over the node caps of several second-tier sizes above their own (2047).  One worker,
    three workers, split and unsplit must agree window for window, and some window of contig 1 that a second tier of
    its own size leaves unpolished for its node count (the single-device call on contig 1 alone) must be polished."""
    from racon_gpu_b200 import api
    import test_overlap_units as tu
    deep = synth_overlap_set(14, contig_lengths=(1600,), depth=170, long_insertions=0.03)
    deep = {k: deep[k] for k in polish_args(deep)}
    noisy = synth_overlap_set(7, contig_lengths=(3000,), depth=600, read_len=(400, 600), long_insertions=0.04)
    noisy = {k: noisy[k] for k in polish_args(noisy)}
    s = _join(deep, noisy)
    kw = dict(window_length=W, quality_threshold=THR, mem_per_poa_batch=1 << 30, deep_windows=True, export_layers=True,
              **SCORES)
    # the smallest aligner budget every window fits, and a bit more: contig 1 in several units
    cols = _planner_columns(s)
    ks = tu.by_contig(cols)
    lo, hi = tu.spans(cols)
    fw = tu.first_windows(cols)
    need = max(tu.min_budget(emu, cols, [k for k in ks[c] if lo[k] <= x <= hi[k]])
               for c in range(2) for x in range(int(fw[c + 1] - fw[c])))
    small = int(need * 1.3)
    want = api.polish_overlaps(**s, devices=[0], aligner_mem=2 << 30, **kw)
    assert want[3]["rounds"] == 1 and want[3]["tier2_windows"] > 0
    for devices in ([0], [0, 0], [0, 0, 0]):
        got = api.polish_overlaps(**s, devices=devices, aligner_mem=small, **kw)
        assert got[3]["split_contigs"] >= 1 and got[3]["rounds"] >= 3, got[3]
        _same(want, got)
    # the edge is reached: node-count failures at 1023 bases that a larger size polishes
    alone, ap, ast, ainfo = api.polish_overlaps(**noisy, **kw)
    first = int(fw[1])
    capped = np.flatnonzero(ast == 4)  # B200POA_NODE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE
    assert capped.size > 0, ast
    assert want[1][first + capped].any(), (ast, want[2][first:])
