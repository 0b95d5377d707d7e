"""GPU: polishing from aligned overlaps on the device (b200poa_polish_overlaps / racon_b200::polish_overlaps) against
racon's host path (breaking points, the window loop of src/polisher.cpp:384-457 into a window arena,
b200poa_polisher_polish_arena) on seeded overlap sets over several contigs, in one and in several rounds, with POA
batches fed in several fills from one aligner batch; a contig too large for the aligner batch is reported; and the
lambda-phage sample reproduces racon's golden edit distances."""
import numpy as np
import pytest

from common import contig_edit_distance, lambda_fixture, lambda_reference
from overlap_cases import host_windows, polish_args, synth_overlap_set
from test_layer_cut import lambda_overlaps

pytestmark = pytest.mark.gpu
W, THR, SCORES = 500, 10.0, {"match": 5, "mismatch": -4, "gap": -8}


#: seed -> the set's arguments.  Seed 14 is deep: windows of more than 200 layers and layers longer than 1023 bases
#: (reads with long insertions), so the driver's dropped-layer branch and its status choice run.
SETS = {11: {}, 12: {}, 14: dict(contig_lengths=(1600, 0, 1200), depth=170, long_insertions=0.03)}


@pytest.mark.parametrize("seed", list(SETS))
@pytest.mark.parametrize("with_t_qual", [True, False])
def test_device_path_equals_host_path(seed, with_t_qual):
    from racon_gpu_b200 import api
    deep = bool(SETS[seed])
    s = synth_overlap_set(seed, **SETS[seed])
    arena = host_windows(s, W, THR, with_t_qual=with_t_qual)
    pol = api.Polisher(devices=[0], batches_per_device=1, mem_per_batch=2 << 30, **SCORES)
    hc, hl, hp, hs = pol.polish_arena(arena, stride=4096)
    pol.close()
    want = api.consensus_list(hc, hl)
    n_win = arena.n_windows
    arena.close()
    if deep:  # windows dropped for depth and for length, and polished ones
        assert (hs == api.EXCEEDED_MAXIMUM_SEQUENCES_PER_POA).any() and (hs == api.EXCEEDED_MAXIMUM_SEQUENCE_SIZE).any()
        assert hp.sum() > 0
    else:
        assert hp.sum() > n_win // 2 and (~hp).sum() > 0  # polished windows, and backbones (contig without overlaps)
    rounds = set()
    # one round; several rounds (a small aligner batch); several fills of two POA batches from one aligner batch
    configs = ((0, 1, 0), (4 << 20, 2, 3), (5 << 20, 2, 1), (6 << 20, 1, 2))
    if deep:  # its contigs do not fit the small aligner batches: one round, POA batches filled once and in several
        configs = ((0, 1, 0), (0, 2, 3))
    for aligner_mem, batches, per_batch in configs:
        got, gp, gs, info = api.polish_overlaps(**polish_args(s, with_t_qual), window_length=W, quality_threshold=THR,
                                                aligner_mem=aligner_mem, poa_batches=batches,
                                                mem_per_poa_batch=1 << 30, max_windows_per_batch=per_batch, **SCORES)
        assert len(got) == n_win
        assert got == want and (gp == hp).all() and (gs == hs).all(), (aligner_mem, batches, per_batch)
        rounds.add(info["rounds"])
    assert min(rounds) == 1 and (deep or max(rounds) >= 2), rounds


def test_contig_too_large_for_the_aligner_batch_is_reported():
    from racon_gpu_b200 import api
    s = synth_overlap_set(13, contig_lengths=(500, 30000), depth=40, read_len=(300, 500))
    with pytest.raises(RuntimeError, match="contig 1 does not fit"):
        api.polish_overlaps(**polish_args(s), window_length=W, quality_threshold=THR, aligner_mem=4 << 20,
                            mem_per_poa_batch=1 << 30, **SCORES)


@pytest.mark.parametrize("case,golden", [("fastq_500", 1312), ("fasta_500", 1566)])
def test_polish_overlaps_lambda_like_racon(oracle, case, golden):
    from racon_gpu_b200 import api
    b, cons, polished, p = lambda_fixture(case)
    ov = lambda_overlaps(case)
    contig = b"".join(b.bases[b.seq_off[s]:b.seq_off[s + 1]].tobytes() for s in b.win_seq_off[:-1])
    q = np.frombuffer(b"".join(o["q"] for o in ov), np.uint8).copy()
    q_off = np.concatenate([[0], np.cumsum([len(o["q"]) for o in ov])]).astype(np.int64)
    qual = np.frombuffer(b"".join(o["qual"] if o["qual"] is not None else b"!" * len(o["q"]) for o in ov), np.uint8)
    got, gp, gs, info = api.polish_overlaps(
        np.frombuffer(contig, np.uint8), np.asarray([0, len(contig)]), None, np.zeros(len(ov), np.int32),
        np.asarray([o["t_begin"] for o in ov]), np.asarray([o["t_begin"] + len(o["t"]) for o in ov]), q, q_off, qual,
        np.asarray([o["qual"] is not None for o in ov], np.uint8), np.asarray([o["q_first"] for o in ov]),
        window_length=p["window_length"], quality_threshold=10.0, match=p["m"], mismatch=p["x"], gap=p["g"],
        tgs=p["tgs"], trim=p["trim"], mem_per_poa_batch=2 << 30)
    assert (gp == polished).all() and got == cons
    assert contig_edit_distance(oracle, got, lambda_reference()) == golden
    assert info["rounds"] == 1
