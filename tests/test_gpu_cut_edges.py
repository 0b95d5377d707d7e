"""GPU: the device layer cut (racon_gpu_b200/csrc/layer_cut.cuh) and the POA batch's gather of its layers
(b200poa_batch_add_windows_from_aligner, poa_gather_kernel) layer for layer against racon's window loop restated
(cut_cases.racon_layers), at every edge: the length and quality filters at their thresholds, empty spans, FASTA and
FASTQ reads, windows per scan thread above 1, window ranges that do not start at 0, adds in chunks, the gathered bytes
and weights, and the POA batch's limits (too deep, too long, batch full) against the host-staged add of the same
windows."""
import numpy as np
import pytest

from cut_cases import edge_set, limits_set, racon_layers, spread_set, weight_set

pytestmark = pytest.mark.gpu
SCORES = {"match": 3, "mismatch": -5, "gap": -4}
#: (window length, quality threshold): 0.02 * w exactly 10 and 10.02; a threshold a mean reaches exactly, one it
#: reaches only after rounding (101 / 10), 0 and a negative one; and w = 50, where one-column layers pass the length
#: filter and only Window::add_layer's empty-span check drops them
EDGES = [(500, 10.0), (501, 10.0), (500, 10.1), (500, 0.0), (500, -1.0), (50, 10.0)]
MODES = ["staged", "staged-chunks", "view", "view-chunks"]
_cache = {}


def _set(kind, *args):
    key = (kind,) + args
    if key not in _cache:
        s = {"edge": edge_set, "spread": spread_set, "weight": weight_set, "limits": limits_set}[kind](*args)
        _cache[key] = (s, s.columns(), _twin_breaking_points(s))
    return _cache[key]


def _aligner(w, threshold=None):
    from racon_gpu_b200.aligner import CUDABatchAligner
    al = CUDABatchAligner(device_id=0, max_gpu_memory=4 << 30)
    al.set_window_length(w, skip_cigars=True)
    if threshold is not None:
        al.set_layer_cut(threshold)
    return al


def _twin_breaking_points(s):
    """The breaking points of a batch without the cut; every overlap without a gap has the planted ones."""
    cols = s.columns()
    al = _aligner(s.w)
    assert al.add_overlaps(cols["q"], cols["q_off"], cols["t"], cols["t_off"], q_first=cols["q_first"],
                           t_begin=cols["t_begin"]) == len(s.ov)
    al.align_all()
    bps = al.breaking_points()
    al.close()
    for k, o in enumerate(s.ov):
        if not o["gapped"]:
            assert (bps[k] == s.planted_breaking_points(k)).all(), k
    return bps


def _add(al, cols, a, b, view):
    added = al.add_overlaps(cols["q"], cols["q_off"][:b + 1], cols["t"], cols["t_off"][:b + 1], first=a,
                            q_first=cols["q_first"], t_begin=cols["t_begin"], view=view,
                            first_window=cols["first_window"], t_length=cols["t_length"],
                            q_quality=cols["q_quality"], has_quality=cols["has_quality"])
    assert added == b - a


def _fills(s, cols, threshold, mode):
    """Run the cut in `mode`; yields (first overlap, last overlap, records, win_lo, counts, device query arena, offset
    of each overlap's read in it) per align_all."""
    n = len(s.ov)
    cuts = [0, n // 3, (2 * n) // 3, n] if mode.endswith("chunks") else [0, n]
    view = mode.startswith("view")
    al = _aligner(s.w, threshold)
    groups = [(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)]
    if not view:  # staged: every chunk added to one batch, then one align_all
        groups = [(0, n, groups)]
    else:  # a view is one add per fill: every chunk is a fill of its own
        groups = [(a, b, [(a, b)]) for a, b in groups]
    for a, b, adds in groups:
        for x, y in adds:
            _add(al, cols, x, y, view)
        al.align_all()
        rec, win_lo, counts = al.layers()
        if view:  # the caller's query column from the fill's first read on
            arena = cols["q"][cols["q_off"][a]:]
            base = cols["q_off"][a:b] - cols["q_off"][a]
        else:  # staged: each pair's query then its target
            arena = np.concatenate([x for k in range(a, b) for x in (cols["q"][cols["q_off"][k]:cols["q_off"][k + 1]],
                                                                     cols["t"][cols["t_off"][k]:cols["t_off"][k + 1]])])
            lens = [(cols["q_off"][k + 1] - cols["q_off"][k]) + (cols["t_off"][k + 1] - cols["t_off"][k])
                    for k in range(a, b)]
            base = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        yield a, b, rec, win_lo, counts, arena, base
        al.reset()
    al.close()


def _check_records(s, cols, bps, threshold, mode):
    """The cut's records equal the restatement applied to the twin's breaking points, field by field, in order."""
    w = s.w
    n_fills = 0
    for a, b, rec, win_lo, counts, arena, base in _fills(s, cols, threshold, mode):
        n_fills += 1
        ov = s.ov[a:b]
        want = racon_layers(ov, bps[a:b], w, threshold)
        lo = int(cols["first_window"][a:b].min())
        hi = int(max(o["first_window"] + (len(s.contigs[o["t_id"]]) + w - 1) // w for o in ov))
        assert (win_lo, len(counts)) == (lo, hi - lo)
        assert counts.tolist() == [len(want.get(lo + i, [])) for i in range(hi - lo)]
        assert (np.diff(rec["window"]) >= 0).all()
        got = {}
        for r in rec:
            k = int(r["overlap"])
            o = ov[k]
            q0 = int(r["q_off"] - base[k]) + o["q_first"]
            ln = int(r["length"])
            got.setdefault(int(r["window"]), []).append((k, q0, ln, int(r["begin"]), int(r["end"]),
                                                         bool(r["has_quality"])))
            i = q0 - o["q_first"]
            assert arena[r["q_off"]:r["q_off"] + ln].tobytes() == o["q"][i:i + ln], (k, q0)
        assert got == want
    assert n_fills == (3 if mode == "view-chunks" else 1)


def _edges_reached(s, bps, threshold):
    """Every planted edge is in the twin's breaking points and the restatement keeps or drops it as it should."""
    w = s.w
    want = racon_layers(s.ov, bps, w, threshold)
    kept = {(x[0], x[2]) for v in want.values() for x in v}  # (overlap, length)
    kept_ov = {x[0] for v in want.values() for x in v}
    tag = {o["tag"]: k for k, o in enumerate(s.ov) if o["tag"]}
    for L in (1, 2, 9, 10, 11, 20):
        for side in ("end", "start"):
            k = tag[f"{side}{L}"]
            pieces = [(int(bps[k][j + 1][1] - bps[k][j][1]), int(bps[k][j + 1][0] - bps[k][j][0]))
                      for j in range(0, bps[k].shape[0], 2)]
            assert (L, L) in pieces  # a layer of L bases over L columns
            assert ((k, L) in kept) == (L >= 0.02 * w and L > 1), (side, L)
    if threshold >= 0:
        assert tag["at"] in kept_ov  # a mean exactly at the threshold
        if "below" in tag:
            assert tag["below"] not in kept_ov
        o = s.ov[tag["at"]]
        assert sum(c - 33 for c in o["qual"]) / len(o["qual"]) == threshold
    assert tag["none"] not in kept_ov and tag["fasta"] in kept_ov and tag["~"] in kept_ov and tag["!~"] in kept_ov
    assert (tag["low"] in kept_ov) == (threshold <= 2)
    fw0, fw1 = s.first_window
    last = fw0 + (len(s.contigs[0]) - 1) // w  # the short last window of contig 0
    assert last in want and max(x[4] for x in want[last]) < len(s.contigs[0]) % w
    assert fw1 in want and fw1 + 1 not in want and fw1 + 2 in want  # an empty window between kept ones


@pytest.mark.parametrize("w,threshold", EDGES)
@pytest.mark.parametrize("mode", MODES)
def test_cut_records_at_the_edges(w, threshold, mode):
    s, cols, bps = _set("edge", w, threshold)
    _edges_reached(s, bps, threshold)
    _check_records(s, cols, bps, threshold, mode)


@pytest.mark.parametrize("n_win", [1, 1023, 1024, 1025, 2049, 10000])
@pytest.mark.parametrize("mode", ["staged", "view-chunks"])
def test_cut_records_window_counts(n_win, mode):
    """The scan kernel with up to ceil(10000 / 1024) = 10 windows per thread, on a window range from 3 on."""
    s, cols, bps = _set("spread", n_win)
    assert s.n_windows == n_win and s.first_window[0] == 3
    want = racon_layers(s.ov, bps, s.w, 10.0)
    assert max(want) == 3 + n_win - 1  # the last window has layers
    _check_records(s, cols, bps, 10.0, mode)


# ------------------------------------------------------------------------------------------------------------------
# the gather
# ------------------------------------------------------------------------------------------------------------------
def _restated_windows(s, bps, threshold, with_t_qual, lo, n_win, weights="quality"):
    """The windows [lo, lo + n_win) as racon builds them from the restated layers, with explicit weights: the
    backbone's quality - 33 (0 for a FASTA target), a layer's quality - 33, or 1 for a read without qualities.
    weights="one" / "plus_one" / "fasta_zero" give the weights a wrong gather would use (for the planted check)."""
    from racon_gpu_b200.windows import WindowBatch
    want = racon_layers(s.ov, bps, s.w, threshold)
    ids = s.window_ids()
    wins, bb_off, bb, bbq = [], [0], [], []
    for win in range(lo, lo + n_win):
        c, a, b = ids[win]
        seq = s.contigs[c][a:b]
        q = s.t_qual[c][a:b] if with_t_qual else None
        bb.append(seq)
        bbq.append(q if q is not None else b"")
        bb_off.append(bb_off[-1] + len(seq))
        bw = np.frombuffer(q, np.uint8).astype(np.int16) - 33 if q is not None else np.zeros(len(seq), np.int16)
        items = [(seq, bw.astype(np.int8), 0, 0)]
        for k, q0, ln, bg, en, has_q in want.get(win, []):
            o = s.ov[k]
            i = q0 - o["q_first"]
            wt = None
            if has_q:
                wt = np.frombuffer(o["qual"][i:i + ln], np.uint8).astype(np.int16) - 33
                wt = {"quality": wt, "one": None, "plus_one": wt + 1, "fasta_zero": wt}[weights]
            elif weights == "fasta_zero":
                wt = np.zeros(ln, np.int16)
            items.append((o["q"][i:i + ln], None if wt is None else wt.astype(np.int8), bg, en))
        wins.append(items)
    batch = WindowBatch.from_lists(wins)
    bb_bases = np.frombuffer(b"".join(bb), np.uint8).copy()
    bb_qual = np.frombuffer(b"".join(bbq), np.uint8).copy() if with_t_qual else None
    return batch, np.asarray(bb_off, np.int64), bb_bases, bb_qual


def _gather_run(kind, *args, threshold, with_t_qual=True):
    """Cut (staged, one add), then one POA batch with consensus and MSA filled by add_windows_from_aligner; the same
    windows restated and staged from the host.  Returns the device's and the host's outputs and the restated batch."""
    from racon_gpu_b200 import api
    s, cols, bps = _set(kind, *args)
    al = _aligner(s.w, threshold)
    _add(al, cols, 0, len(s.ov), False)
    al.align_all()
    _, lo, counts = al.layers()
    batch, bb_off, bb, bbq = _restated_windows(s, bps, threshold, with_t_qual, lo, len(counts))
    assert (np.diff(batch.win_seq_off) - 1 == counts).all()
    dev = api.PoaBatch(max_gpu_mem=2 << 30, output_mask=api.OUTPUT_CONSENSUS | api.OUTPUT_MSA, **SCORES)
    n, seqs_added = dev.add_windows_from_aligner(al, bb_off, bb, bbq)
    assert n == batch.n_windows and (seqs_added == counts).all()
    dev.generate_poa()
    dc, dv, dst = dev.get_consensus()
    msa, mst = dev.get_msa()
    host = api.PoaBatch(max_gpu_mem=2 << 30, **SCORES)
    assert host.add_windows(batch)[0] == batch.n_windows
    host.generate_poa()
    hc, hv, hst = host.get_consensus()
    dev.close()
    host.close()
    al.close()
    return s, bps, batch, (dc, dv, dst, msa, mst), (hc, hv, hst)


GATHER_SETS = [("edge", w, thr) for w, thr in EDGES] + [("weight", False, 0.0), ("weight", True, 0.0)]


def _gather_case(case):
    kind, arg, thr = case
    if kind == "weight":  # arg: a FASTA target
        return _gather_run("weight", arg, threshold=thr, with_t_qual=not arg)
    return _gather_run("edge", arg, thr, threshold=thr)


@pytest.mark.parametrize("case", GATHER_SETS, ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}")
def test_gathered_bytes_spell_the_layers(case):
    """Every MSA row without its gaps spells its sequence: the backbone first, then the layers in
    b200poa_layer_order -- the bytes the gather copied from the aligner's arena."""
    from racon_gpu_b200 import api
    _, _, batch, (dc, dv, dst, msa, mst), _ = _gather_case(case)
    checked = 0
    for i in range(batch.n_windows):
        seqs, _, begins, _ = batch.window(i)
        order = api.layer_order(begins)
        assert mst[i] == api.SUCCESS and order[0] == 0
        assert [r.replace(b"-", b"") for r in msa[i]] == [seqs[o] for o in order], i
        checked += len(seqs) - 1
    assert checked > 0


@pytest.mark.parametrize("case", GATHER_SETS, ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}")
def test_gathered_weights_equal_oracle_and_host(oracle, case):
    """Consensus and coverage in full band, bit for bit: the oracle fed the restated layers with their explicit
    weights, and a host-staged add_windows of the same windows.  For the weight sets, the consensus with weights
    quality - 33 differs from the one with weight 1, with quality - 32, and with FASTA reads weighing 0, so a wrong
    weight in the gather cannot pass."""
    from racon_gpu_b200 import api
    s, bps, batch, (dc, dv, dst, _, _), (hc, hv, hst) = _gather_case(case)
    assert dc == hc and (dst == hst).all() and all((x == y).all() for x, y in zip(dv, hv))
    m, x, g = SCORES["match"], SCORES["mismatch"], SCORES["gap"]
    oc, ocov, _ = oracle.polish(batch, api.processing_order(batch), m, x, g, tgs=False, trim=False, threads=8,
                                stride=8192)
    nseq = np.diff(batch.win_seq_off)
    deep = np.flatnonzero(nseq >= 3)  # racon leaves a window of fewer than three sequences unpolished
    assert deep.shape[0] > 0
    for i in deep:
        assert dst[i] == api.SUCCESS and dc[i] == oc[i] and (dv[i] == ocov[i]).all(), i
    if case[0] == "weight":
        _, fasta_target, thr = case
        lo = s.first_window[0]
        for wrong in ("one", "plus_one", "fasta_zero"):
            b2 = _restated_windows(s, bps, thr, not fasta_target, lo, batch.n_windows, weights=wrong)[0]
            wc = oracle.polish(b2, api.processing_order(b2), m, x, g, tgs=False, trim=False, threads=8, stride=8192)[0]
            assert any(wc[i] != oc[i] for i in deep), wrong


# ------------------------------------------------------------------------------------------------------------------
# the POA batch's limits and sub-ranges
# ------------------------------------------------------------------------------------------------------------------
def test_gather_limits_and_subranges_equal_host(monkeypatch):
    """A window of more than 200 layers, a layer longer than 1023 bases and a POA batch that fills mid-range: every
    fill of add_windows_from_aligner over [first, last) sub-ranges takes up exactly where the previous one stopped,
    and adds, drops and computes what the host-staged add_windows of the same windows does."""
    from racon_gpu_b200 import api
    monkeypatch.setenv("B200POA_MAX_STAGING_MB", "1")  # a small batch: it fills before the range ends
    s, cols, bps = _set("limits")
    thr = 10.0
    al = _aligner(s.w, thr)
    _add(al, cols, 0, len(s.ov), False)
    al.align_all()
    _, lo, counts = al.layers()
    batch, bb_off, bb, bbq = _restated_windows(s, bps, thr, True, lo, len(counts))
    nseq = np.diff(batch.win_seq_off)
    deep_win, long_win = 7, 12
    assert nseq[deep_win] - 1 > 200
    assert max(len(batch.window(long_win)[0][i]) for i in range(1, nseq[long_win])) > 1023
    dev = api.PoaBatch(max_gpu_mem=1 << 30, **SCORES)
    host = api.PoaBatch(max_gpu_mem=1 << 30, **SCORES)
    cursor, fills, full_stops, seen = 0, 0, 0, {}
    while cursor < batch.n_windows:
        last = batch.n_windows if fills % 2 == 0 else min(batch.n_windows, cursor + 17)
        dev.reset()
        host.reset()
        n, seqs_added = dev.add_windows_from_aligner(al, bb_off, bb, bbq, first=cursor, last=last)
        hn, hseqs = host.add_windows(batch.slice(cursor, last))
        assert n == hn and n > 0 and (seqs_added == hseqs).all(), (cursor, last)
        full_stops += n < last - cursor
        dev.generate_poa()
        host.generate_poa()
        dc, dv, dst = dev.get_consensus()
        hc, hv, hst = host.get_consensus()
        assert dc == hc and (dst == hst).all() and all((x == y).all() for x, y in zip(dv, hv)), cursor
        for i in range(n):
            seen[cursor + i] = int(seqs_added[i])
        cursor += n
        fills += 1
    assert sorted(seen) == list(range(batch.n_windows))
    assert full_stops >= 1 and fills >= 3
    assert seen[deep_win] == 199 and seen[long_win] == nseq[long_win] - 2  # 200 sequences with the backbone
    dev.close()
    host.close()
    al.close()
