"""Seeded overlap sets over several contigs, and racon's host path over them (TEST INFRASTRUCTURE).

`synth_overlap_set` makes contigs, reads drawn from them with errors (either strand, with or without qualities) and the
overlaps racon would keep, in racon's order; `host_path` polishes them the way racon does without the device cut:
breaking points from the aligner, the loop of src/polisher.cpp:384-457 (cut_cases.racon_layers) on the host into a
window arena, then b200poa_polisher_polish_arena."""
import numpy as np

from cut_cases import racon_layers

COMP = bytes.maketrans(b"ACGT", b"TGCA")


def _mutate(rng, s: bytes, e: float) -> bytes:
    out = bytearray()
    for c in s:
        x = rng.random()
        if x < e / 3:
            out.append(b"ACGT"[rng.integers(4)])
        elif x < 2 * e / 3:
            continue
        elif x < e:
            out += bytes([c, b"ACGT"[rng.integers(4)]])
        else:
            out.append(c)
    return bytes(out)


def synth_overlap_set(seed: int, contig_lengths=(3100, 0, 2400, 1750, 4000), depth=6, error=0.08, read_len=(600, 1800),
                      long_insertions=0.0):
    """Columns for api.polish_overlaps.  Contig 1 is empty when its length is 0; a contig may get no overlap.
    long_insertions: the share of reads with 1100 random bases inserted in their middle, which gives the window
    there a layer longer than the POA batch's max_sequence_size (1023)."""
    rng = np.random.default_rng(seed)
    contigs = [rng.choice(np.frombuffer(b"ACGT", np.uint8), size=n).tobytes() for n in contig_lengths]
    t_qual = [bytes(rng.integers(33 + 5, 33 + 40, size=len(c), dtype=np.uint8)) for c in contigs]
    ov = []
    for c, t in enumerate(contigs):
        if len(t) < 400 or c == 3:  # contig 3 has windows but no overlap
            continue
        for _ in range(depth * len(t) // 1000):
            ln = int(rng.integers(*read_len))
            tb = int(rng.integers(0, max(1, len(t) - 200)))
            te = min(len(t), tb + ln)
            seg = _mutate(rng, t[tb:te], error)
            if rng.random() < long_insertions:
                mid = len(seg) // 2
                seg = seg[:mid] + bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), size=1100)) + seg[mid:]
            lead, tail = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), size=int(rng.integers(0, 60)))), b""
            strand = int(rng.integers(2))
            has_q = bool(rng.random() < 0.7)
            qual = bytes(rng.integers(33 + 3, 33 + 30, size=len(lead) + len(seg), dtype=np.uint8)) if has_q else None
            if has_q and rng.random() < 0.2:  # a low-quality read: its layers fail the quality filter
                qual = bytes(rng.integers(33, 33 + 9, size=len(qual), dtype=np.uint8))
            # the strand-adjusted read is lead + seg; racon cuts [q_first, q_first + len(seg)) out of it
            ov.append({"t_id": c, "t_begin": tb, "t_end": te, "q": seg, "q_first": len(lead),
                       "qual": qual[len(lead):] if has_q else None, "strand": strand})
    order = rng.permutation(len(ov))  # racon's order interleaves contigs; the driver partitions it stably
    ov = [ov[i] for i in order]
    t_off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.int64)
    q_off = np.concatenate([[0], np.cumsum([len(o["q"]) for o in ov])]).astype(np.int64)
    return {
        "contigs": contigs, "t_bases": np.frombuffer(b"".join(contigs), np.uint8).copy(), "t_off": t_off,
        "t_qual": np.frombuffer(b"".join(t_qual), np.uint8).copy(), "ov": ov,
        "t_id": np.asarray([o["t_id"] for o in ov], np.int32), "t_begin": np.asarray([o["t_begin"] for o in ov], np.int32),
        "t_end": np.asarray([o["t_end"] for o in ov], np.int32),
        "q_bases": np.frombuffer(b"".join(o["q"] for o in ov), np.uint8).copy(), "q_off": q_off,
        "q_qual": np.frombuffer(b"".join(o["qual"] if o["qual"] else b"!" * len(o["q"]) for o in ov), np.uint8).copy(),
        "has_quality": np.asarray([o["qual"] is not None for o in ov], np.uint8),
        "q_first": np.asarray([o["q_first"] for o in ov], np.int32),
    }


def polish_args(s, with_t_qual=True):
    return dict(t_bases=s["t_bases"], t_off=s["t_off"], t_qual=s["t_qual"] if with_t_qual else None, t_id=s["t_id"],
                t_begin=s["t_begin"], t_end=s["t_end"], q_bases=s["q_bases"], q_off=s["q_off"], q_qual=s["q_qual"],
                has_quality=s["has_quality"], q_first=s["q_first"])


def host_windows(s, w: int, threshold: float, with_t_qual=True, device=0):
    """racon's host path up to the windows: breaking points from the aligner (no cut), then polisher.cpp:384-457 into
    a window arena (b200poa_arena_*).  Returns the finalized WindowArena."""
    from racon_gpu_b200 import api
    from racon_gpu_b200.aligner import CUDABatchAligner
    al = CUDABatchAligner(device_id=device, max_gpu_memory=4 << 30)
    al.set_window_length(w, skip_cigars=True)
    ov = s["ov"]
    t_seg = [s["contigs"][o["t_id"]][o["t_begin"]:o["t_end"]] for o in ov]
    t = np.frombuffer(b"".join(t_seg), np.uint8).copy()
    t_off = np.concatenate([[0], np.cumsum([len(x) for x in t_seg])]).astype(np.int64)
    bps, done = [], 0
    while done < len(ov):
        done += al.add_overlaps(s["q_bases"], s["q_off"], t, t_off, first=done, q_first=s["q_first"],
                                t_begin=s["t_begin"])
        al.align_all()
        bps += al.breaking_points()
        al.reset()
    al.close()
    arena = api.WindowArena()
    first_window = []
    for c, contig in enumerate(s["contigs"]):
        first_window.append(arena.n_windows)
        for j in range(0, len(contig), w):
            bb = contig[j:j + w]
            q = s["t_qual"][s["t_off"][c] + j:s["t_off"][c] + j + len(bb)].tobytes() if with_t_qual else b"!" * len(bb)
            arena.add_window(bb, q)
    for win, layers in sorted(racon_layers([dict(o, first_window=first_window[o["t_id"]]) for o in ov], bps, w,
                                           threshold).items()):
        for k, q0, ln, bg, en, has_q in layers:
            o = ov[k]
            data = o["q"][q0 - o["q_first"]:q0 - o["q_first"] + ln]
            qq = o["qual"][q0 - o["q_first"]:q0 - o["q_first"] + ln] if has_q else None
            assert arena.add_layer(win, data, qq, bg, en)
    arena.finalize(view=False)
    return arena
