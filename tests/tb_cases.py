"""The POA traceback at its edges: window sets, what each must reach in the emulation's traceback report, and checks.

traceback() in racon_gpu_b200/csrc/poa_core.cuh walks the alignment through a 64-row x 32-column tile of the score
matrix and falls back to other paths at the tile's edges: a re-anchored tile, steps read from global memory (more than
32 in-edges, CSR entries past TB_PRED_CAP, a predecessor still below a re-anchored tile), NEG-filled chunks outside the
band, the adaptive band's edge test, the row-0 tail, the 32-entry output buffer and, on 32-bit cells, traceback_i32().

Every case is a list of runs (fill_cases.run: one batch configuration over one window set).  The CPU suite runs each
through the emulation, which walks a scalar twin after every traceback and reports which paths were taken; every case
must reach what its name promises (tb_reach_failures) and, in full band, every alignment must equal spoa's (the
oracle's poa_oracle_alignment_digests) (tests/test_tb_reach.py).  The GPU suite runs the same batches on the digest
build and compares per-read alignment digests with the emulation and the oracle (tests/test_gpu_traceback.py).
"""
from __future__ import annotations

import numpy as np

import fill_cases as fc
from fill_cases import ACGT, GB, _window, run
from racon_gpu_b200.windows import WindowBatch, synth_windows

#: insertion lengths of far_preds: the junction row's other predecessor lies length + 1 rows back, and a tile
#: re-anchored at the junction holds rows down to 63 rows back
FAR_INSERTIONS = (62, 63, 64, 65, 66, 100)
#: random prefixes of the ends case: row-0 tails of these lengths
PREFIXES = (1, 31, 32, 33, 64, 100)
#: scorings with many equal-score paths, and fill_cases' three that switch from int16 to 32-bit cells in a window
TIE_SCORINGS = ((127, -1, 0), (0, -1, -1), (2, 1, -1), (1, -1, -1)) + fc.SWITCHING


def far_pred_windows(depth: int = 8) -> WindowBatch:
    """One window per FAR_INSERTIONS length: every other read carries that many Ns after backbone position 149, the
    others are the backbone itself.  The graph's ranks put the insertion between backbone nodes 149 and 150.  (An
    insertion of ACGT bases does not stay in one piece: with linear gaps, bases of it that match the backbone nearby
    give equal-score alignments that split it.)"""
    rng = np.random.default_rng(31)
    wins = []
    for n in FAR_INSERTIONS:
        truth = rng.choice(ACGT, 300).tobytes()
        ins = b"N" * n
        reads = [truth[:150] + ins + truth[150:] if i % 2 == 0 else truth for i in range(depth)]
        wins.append(_window([truth] + reads, [None] * (depth + 1)))
    return WindowBatch.from_lists(wins)


HUBS = ((300, 40), (320, 80), (340, 120))  # (backbone position, reads whose deletion ends there)


def hub_windows() -> WindowBatch:
    """Windows with three hubs within 40 ranks (HUBS): n reads lack 1..n bases ending at the hub's position.  A read
    aligned after others reuses an earlier read's skip edge when that is cheaper than its own deletion, so a hub gets
    fewer than n + 1 in-edges: 40 and 26 at most in these two windows, so that one of them has a row past the 32 in-edges
    a tile step handles."""
    rng = np.random.default_rng(32)
    wins = []
    for w in range(2):
        truth = rng.choice(ACGT, 500).tobytes()
        reads = [truth[:h - k] + truth[h:] for h, n in HUBS for k in range(1, n + 1)]
        reads = [reads[i] for i in rng.permutation(len(reads))]
        wins.append(_window([truth] + reads, [None] * (len(reads) + 1)))
    return WindowBatch.from_lists(wins)


def prefix_windows(depth: int = 6) -> WindowBatch:
    """One window per PREFIXES length: every read is the backbone behind a random prefix of that many bases."""
    rng = np.random.default_rng(33)
    wins = []
    for n in PREFIXES:
        truth = rng.choice(ACGT, 300).tobytes()
        reads = [rng.choice(ACGT, n).tobytes() + truth for _ in range(depth)]
        wins.append(_window([truth] + reads, [None] * (depth + 1)))
    return WindowBatch.from_lists(wins)


def missing_end_windows(depth: int = 8) -> WindowBatch:
    """Reads that lack the first or the last 40-150 backbone bases but span (0, L - 1), so that they are aligned to
    the whole graph: long runs of vertical moves at both ends of the walk.
    The reads' differences from the backbone (substitutions) lie in the middle: an error near a read's end would add a
    source node or a sink close to it, and the walk would leave the graph through that shortcut instead."""
    rng = np.random.default_rng(34)
    wins = []
    for w in range(4):
        truth = rng.choice(ACGT, 400).tobytes()
        reads = []
        for i in range(depth):
            a = np.frombuffer(truth, dtype=np.uint8).copy()
            hit = np.flatnonzero(rng.random(80) < 0.05) + 160
            a[hit] = rng.choice(ACGT, hit.shape[0])
            k = int(rng.integers(40, 151))
            reads.append(a[k:].tobytes() if i % 2 == 0 else a[:400 - k].tobytes())
        wins.append(_window([truth] + reads, [None] * (depth + 1)))
    return WindowBatch.from_lists(wins)


def ends_windows() -> WindowBatch:
    return fc.concat(prefix_windows(), missing_end_windows())


def tie_batch(sc) -> WindowBatch:
    """fill_cases' scoring windows: switching scorings get reads just around the length at which int16 stops being
    provably enough."""
    L = {fc.SWITCHING[0]: 450, fc.SWITCHING[1]: 262, fc.SWITCHING[2]: 350}.get(sc, 200)
    return synth_windows(3, L, 16, 0.15, seed=27)


def adaptive_windows() -> WindowBatch:
    from test_emu import deletion_windows
    return fc.concat(deletion_windows(n=4), fc.short_deletion_windows(), synth_windows(4, 500, 16, 0.12, seed=26))


def band_edge_windows() -> WindowBatch:
    from test_emu import deletion_windows
    return fc.concat(deletion_windows(n=4), fc.long_read_windows())


def cases():
    from common import partial_span_windows
    out = {}
    ladder = fc.ladder_of_lengths()
    out["tile_edges"] = [run("tile_edges_full", ladder, msz=1279, mem=4 * GB),
                         run("tile_edges_static256", ladder, mode="static", msz=1279, mem=4 * GB)]
    far = far_pred_windows()
    out["far_preds"] = [run("far_preds_full", far), run("far_preds_static256", far, mode="static")]
    hubs = fc.concat(fc.deep_windows(), hub_windows())
    out["hubs"] = [run("hubs_full", hubs, msz=2047, depth=256),
                   run("hubs_static256", hubs, mode="static", msz=2047, depth=256)]
    ends = ends_windows()
    out["ends"] = [run("ends_full", ends), run("ends_static256", ends, mode="static")]
    edges = band_edge_windows()
    out["band_edges"] = [run(f"band_edges_static{w}", edges, mode="static", band=w) for w in (64, 128, 256)]
    adapt = adaptive_windows()
    out["adaptive"] = [run(f"adaptive{w}", adapt, mode="adaptive", band=w) for w in (64, 128)]
    out["ties"] = [run("ties_%d_%d_%d" % sc, tie_batch(sc), scoring=sc) for sc in TIE_SCORINGS]
    part = partial_span_windows(n=6)
    out["partial"] = [run("partial_full", part), run("partial_static256", part, mode="static")]
    odd = fc.odd_letter_windows()
    out["letters"] = [run("letters_full", odd), run("letters_static256", odd, mode="static")]
    return out


def tb_reach_failures(case: str, r, out) -> list:
    """What run r of `case` must reach, from the emulation's reports (fill_cases.emu_run); returns the unmet promises."""
    b = r["batch"]
    rep, fill = out["tb_reach"], out["reach"]
    tot = {k: int(v.sum()) for k, v in rep.items()}
    need = []
    fills = int(out["count"].sum())
    if tot["tracebacks"] != fills:  # the twin checked the traceback of every fill, adaptive tries included
        need.append(f"a twin check after each of the {fills} fills, got {tot['tracebacks']}")
    if tot["twin_mismatches"]:
        need.append(f"no traceback that differs from its scalar twin, got {tot['twin_mismatches']}")
    if case == "tile_edges":  # (10 % error at depth 5 never puts a predecessor below a tile: no re-anchor here)
        for k in ("count_mod0", "count_mod1", "count_mod31"):
            if tot[k] == 0:
                need.append(k)
    elif case == "far_preds":
        for w, n in enumerate(FAR_INSERTIONS):
            far = int(rep["global_far"][w])
            if n >= 63 and far == 0:  # predecessor n + 1 >= 64 rows back: below a tile re-anchored at the junction
                need.append(f"window {w} (insertion {n}): global steps for a predecessor more than 63 rows back")
            if n == 62 and far != 0:  # 63 rows back: inside the re-anchored tile
                need.append(f"window {w} (insertion {n}): no global step for a predecessor 63 rows back, got {far}")
        if tot["reanchors"] == 0:
            need.append("reanchors")
    elif case == "hubs":
        # (no window here puts more than TB_PRED_CAP entries into one tile: global_pred_cap is not reached)
        nh = hub_windows().n_windows
        if rep["global_npred"][-nh:].sum() == 0 or tot["global_npred"] == 0:
            need.append("global steps of rows with more than 32 in-edges, in a hub window and overall")
    elif case == "ends":
        npre = len(PREFIXES)
        for w, n in enumerate(PREFIXES):
            if n >= 32 and rep["row0_tail32"][w] == 0:
                need.append(f"window {w}: a row-0 tail of {n}")
            if n >= 64 and rep["row0_tail64"][w] == 0:
                need.append(f"window {w}: a row-0 tail of {n} (64 or more)")
        if (rep["vrun32"][npre:] == 0).any():
            need.append("vertical runs of 32 or more in every missing-end window")
    elif case == "band_edges":
        if tot["neg_chunk_steps"] == 0:
            need.append("steps that read NEG-filled chunks")
    elif case == "adaptive":
        if tot["band_hits"] == 0 or fill["retries_full"].sum() == 0:
            need.append("band_hit and retries up to the full matrix")
    elif case == "ties":
        sc = r["scoring"]
        if sc in fc.SWITCHING and not ((rep["i32_reads"] > 0) & (rep["i32_reads"] < np.diff(b.win_seq_off) - 1)).any():
            need.append("traceback_i32 and the tile walk in one window")
        if sc not in fc.SWITCHING and tot["i32_reads"]:
            need.append("int16 cells only")
    elif case == "partial":
        if tot["partial_reads"] == 0:
            need.append("tracebacks against subgraphs")
    elif case == "letters":
        if (fill["dyn_rows"] == 0).any():
            need.append("letters outside ACGT in every window")
    return need


def mismatch_report(r, out) -> list:
    """The emulation's first twin mismatch per window, as text."""
    bad = []
    for w, m in enumerate(out["tb_mismatch"]):
        if m[0] >= 0:
            rd, tr, k, tn, tp, en, ep, tc, ec = (int(v) for v in m)
            bad.append(f"{r['name']}: window {w} read {rd} try {tr}: entry {k} of {ec} is ({en}, {ep}), the scalar twin's "
                       f"entry {k} of {tc} is ({tn}, {tp})")
    return bad


def oracle_aln(oracle, r):
    """spoa's alignment digests and entry counts of the run's windows (full band only)."""
    from racon_gpu_b200 import api
    m, x, g = r["scoring"]
    dg, cnt = oracle.alignment_digests(r["batch"], api.processing_order(r["batch"]), m, x, g)
    return {"aln_digest": dg, "aln_count": cnt}
