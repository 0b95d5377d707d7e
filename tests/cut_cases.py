"""racon's window-layer loop restated, and overlap sets that reach the device layer cut's edges (TEST INFRASTRUCTURE).

`racon_layers` is the one plain restatement of src/polisher.cpp:403-457 the suite checks the cut against (the host build
in tests/test_layer_cut.py, the host window arena in tests/overlap_cases.py, the device cut and gather in
tests/test_gpu_cut_edges.py)."""
import numpy as np


def racon_layers(ov, bps, w, threshold):
    """src/polisher.cpp:403-457 restated: per window id, the layers Window::add_layer keeps, in racon's add order
    (overlap, then breaking-point pair), as (overlap, q0, length, begin, end, has_quality).

    ov[k] needs "qual" (the read's qualities from q_first on, or None), "q_first" and "first_window" (the contig's
    id_to_first_window_id); bps[k] is its (n, 2) array of (t, q) breaking points.  Followed literally: the length filter
    compares q1 - q0 with 0.02 * w as doubles; the quality filter is a running double sum of quality - 33, one division
    and "<"; Window::add_layer drops an empty span (src/window.cpp:45-47)."""
    out = {}
    for k, (o, bp) in enumerate(zip(ov, bps)):
        for j in range(0, bp.shape[0], 2):
            (t0, q0), (t1, q1) = (int(x) for x in bp[j]), (int(x) for x in bp[j + 1])
            if q1 - q0 < 0.02 * w:
                continue
            if o["qual"] is not None:
                avg = 0.0
                for c in o["qual"][q0 - o["q_first"]:q1 - o["q_first"]]:
                    avg += c - 33
                avg /= q1 - q0
                if avg < threshold:
                    continue
            start = (t0 // w) * w
            if t0 - start == t1 - start - 1:
                continue
            out.setdefault(o["first_window"] + t0 // w, []).append((k, q0, q1 - q0, t0 - start, t1 - start - 1,
                                                                     o["qual"] is not None))
    return out


# ------------------------------------------------------------------------------------------------------------------
# overlap sets for the device cut: reads are copies of a contig segment with substitutions only, so edlib's path is
# all matches and mismatches and every breaking point is known by construction
# ------------------------------------------------------------------------------------------------------------------
ACGT = b"ACGT"


def _contig(rng, n):
    return rng.choice(np.frombuffer(ACGT, np.uint8), size=n).tobytes()


def _subst(rng, seg: bytes, spacing: int = 24) -> bytes:
    """seg with isolated substitutions (at least `spacing` apart): one substitution costs 1 and any path with an
    insertion and a deletion at least 2, so the alignment is unique and has no gap."""
    out = bytearray(seg)
    i = int(rng.integers(spacing // 2, spacing))
    while i < len(out):
        out[i] = ACGT[(ACGT.index(out[i]) + int(rng.integers(1, 4))) % 4]
        i += int(rng.integers(spacing, 2 * spacing))
    return bytes(out)


def _qual_sum(n: int, s: int) -> bytes:
    """n qualities whose (quality - 33) add up to exactly s"""
    base, extra = divmod(s, n)
    return bytes([33 + base + 1] * extra + [33 + base] * (n - extra))


class OverlapSet:
    """Contigs (each with its first window id) and overlaps on them, in racon's order; `columns` gives the aligner's
    inputs."""

    def __init__(self, w, first_window=0):
        self.w = w
        self.contigs, self.t_qual, self.first_window, self.ov = [], [], [], []
        self.next_window = first_window

    def contig(self, seq: bytes, qual: bytes) -> int:
        self.contigs.append(seq)
        self.t_qual.append(qual)
        self.first_window.append(self.next_window)
        self.next_window += (len(seq) + self.w - 1) // self.w
        return len(self.contigs) - 1

    def read(self, rng, c, tb, te, qual, seg=None, tag=None, gapped=False):
        """Overlap of contig c's [tb, te): the read is seg (default: the contig's bases with substitutions); qual: the
        qualities of seg (None: a FASTA read).  A random lead sits before q_first in the strand-adjusted read.
        gapped: seg has insertions, so its breaking points are not known by construction."""
        seg = _subst(rng, self.contigs[c][tb:te]) if seg is None else seg
        assert qual is None or len(qual) == len(seg)
        self.ov.append({"t_id": c, "t_begin": tb, "t_end": te, "q": seg, "q_first": int(rng.integers(0, 40)),
                        "qual": qual, "first_window": self.first_window[c], "tag": tag, "gapped": gapped})
        return len(self.ov) - 1

    def planted_breaking_points(self, k):
        """Overlap k's breaking points when its alignment has no gap (Overlap::find_breaking_points_from_cigar on an
        all-match path): per window it touches, its first column and one past its last, with the read's positions."""
        o = self.ov[k]
        tb, te, qf, out = o["t_begin"], o["t_end"], o["q_first"], []
        a = tb
        while a < te:
            b = min(te, (a // self.w + 1) * self.w)
            out += [(a, qf + a - tb), (b, qf + b - tb)]
            a = b
        return np.asarray(out, dtype=np.uint32).reshape(-1, 2)

    @property
    def n_windows(self):
        return self.next_window - self.first_window[0]

    def window_ids(self):
        """window id -> (contig, start, end) of every window of the set's contigs"""
        out = {}
        for c, t in enumerate(self.contigs):
            for j in range(0, len(t), self.w):
                out[self.first_window[c] + j // self.w] = (c, j, min(j + self.w, len(t)))
        return out

    def columns(self):
        ov = self.ov
        q = np.frombuffer(b"".join(o["q"] for o in ov), np.uint8).copy()
        t_seg = [self.contigs[o["t_id"]][o["t_begin"]:o["t_end"]] for o in ov]
        t = np.frombuffer(b"".join(t_seg), np.uint8).copy()
        q_off = np.concatenate([[0], np.cumsum([len(o["q"]) for o in ov])]).astype(np.int64)
        t_off = np.concatenate([[0], np.cumsum([len(x) for x in t_seg])]).astype(np.int64)
        qual = np.frombuffer(b"".join(o["qual"] if o["qual"] is not None else b"!" * len(o["q"]) for o in ov),
                             np.uint8).copy()
        return {"q": q, "q_off": q_off, "t": t, "t_off": t_off, "q_quality": qual,
                "has_quality": np.asarray([o["qual"] is not None for o in ov], np.uint8),
                "q_first": np.asarray([o["q_first"] for o in ov], np.int32),
                "t_begin": np.asarray([o["t_begin"] for o in ov], np.int32),
                "first_window": np.asarray([o["first_window"] for o in ov], np.int64),
                "t_length": np.asarray([len(self.contigs[o["t_id"]]) for o in ov], np.int32)}


def _good(rng, n):
    return bytes(rng.integers(33 + 25, 33 + 41, size=n, dtype=np.uint8))


def edge_set(w: int, threshold: float, seed: int = 1) -> OverlapSet:
    """The cut's edges, planted through real alignments (tests/test_gpu_cut_edges.py asserts each is reached):
    layers of 1, 2, 9, 10, 11 and 20 bases at the start and the end of overlaps (0.02 * w, one-column spans begin ==
    end, end == begin + 1); a layer whose mean quality is exactly the threshold and one a quality point lower; FASTA
    reads among FASTQ reads; qualities '!' and '~'; an overlap that keeps no layer; the short last window of a contig;
    an empty window between kept ones.  The first contig starts at window 5, so the batch's window range starts there."""
    rng = np.random.default_rng(seed)
    s = OverlapSet(w, first_window=5)
    c0 = s.contig(_contig(rng, 6 * w + w // 3 + 7), _good(rng, 6 * w + w // 3 + 7))
    c1 = s.contig(_contig(rng, 3 * w), _good(rng, 3 * w))
    n0 = len(s.contigs[c0])
    for L in (9, 10, 11):  # layers of L bases at the end of an overlap (window 1) and at its start (window 3)
        s.read(rng, c0, w - w // 2, w + L, _good(rng, w // 2 + L), tag=f"end{L}")
        s.read(rng, c0, 4 * w - L, 4 * w + w // 2, _good(rng, L + w // 2), tag=f"start{L}")
    for L in (1, 2, 20):
        s.read(rng, c0, 2 * w - w // 2, 2 * w + L, _good(rng, w // 2 + L), tag=f"end{L}")
        s.read(rng, c0, 3 * w - L, 3 * w + w // 2, None, tag=f"start{L}")
    # one layer of n_q bases per overlap (window 4), mean quality exactly the threshold and one quality point lower
    n_q = w - w % 10
    at = max(0, round(threshold * n_q))
    s.read(rng, c0, 5 * w - n_q, 5 * w, _qual_sum(n_q, at), tag="at")
    if at > 0:
        s.read(rng, c0, 5 * w - n_q, 5 * w, _qual_sum(n_q, at - 1), tag="below")
    # FASTA and FASTQ reads over several windows; qualities '!' and '~'
    s.read(rng, c0, 0, 3 * w - 17, None, tag="fasta")
    s.read(rng, c0, 13, 3 * w + 40, (b"!~" * (2 * w))[:3 * w + 27], tag="!~")
    s.read(rng, c0, w + 3, 4 * w - 5, b"~" * (3 * w - 8), tag="~")
    s.read(rng, c0, 2, 2 * w + 60, _good(rng, 2 * w + 58))
    # an overlap that keeps no layer: two one-column spans across a window boundary
    s.read(rng, c0, 2 * w - 1, 2 * w + 1, _good(rng, 2), tag="none")
    # a read whose layers are all below a threshold of 10 (kept at 0 and below)
    s.read(rng, c0, w + 40, 3 * w - 40, b"#" * (2 * w - 80), tag="low")
    # the short last window
    s.read(rng, c0, 5 * w - 30, n0, _good(rng, n0 - 5 * w + 30))
    s.read(rng, c0, 4 * w + 11, n0 - 3, None)
    # contig 1: windows 0 and 2 kept, window 1 empty between them
    s.read(rng, c1, 10, w - 5, _good(rng, w - 15))
    s.read(rng, c1, 2 * w + 3, 3 * w, None)
    s.read(rng, c1, 2 * w + 20, 3 * w - 2, _good(rng, w - 22))
    return s


def spread_set(n_win: int, w: int = 500, seed: int = 1) -> OverlapSet:
    """One contig of n_win windows (the last one short), from window 3 on, with short overlaps spread thinly over it:
    the cut's scan runs with ceil(n_win / 1024) windows per thread."""
    rng = np.random.default_rng(seed + n_win)
    s = OverlapSet(w, first_window=3)
    n = n_win * w - 7
    c = s.contig(_contig(rng, n), _good(rng, n))
    starts = sorted(set([0, max(0, n - w)] + [int(x) for x in rng.integers(0, n, size=60)] +
                        [min(n - 1, k * w - 20) for k in (1023, 1024, 1025, 2048, 2049) if k * w - 20 < n]))
    for tb in starts:
        te = min(n, tb + int(rng.integers(40, 2 * w)))
        s.read(rng, c, tb, te, _good(rng, te - tb) if rng.random() < 0.7 else None)
    return s


def weight_set(fasta_target: bool, seed: int = 1) -> OverlapSet:
    """Windows whose consensus the weights decide: at 20 columns a minority of reads carries one base and a majority
    another, and only the weights quality - 33 pick the minority's.  Window 0: one read of quality '$' (weight 3)
    against five of '!' (0); window 1: the same read against five FASTA reads (weight 1 each, so the majority wins);
    window 2: one read of '~' (93) against five of '!'; window 3: three reads of '5' (20) against five of '#' (2).
    Every read covers its window; the target's qualities are '"' (weight 1), or none (a FASTA target, weight 0).
    For a quality threshold of 0: the reads of '!' have a mean exactly at it."""
    rng = np.random.default_rng(seed)
    w = 500
    s = OverlapSet(w, first_window=2)
    t = _contig(rng, 5 * w)
    c = s.contig(t, None if fasta_target else b'"' * len(t))
    groups = [((1, b"$"), (5, b"!")), ((1, b"$"), (5, None)), ((1, b"~"), (5, b"!")), ((3, b"5"), (5, b"#"))]
    for j, ((n_a, q_a), (n_b, q_b)) in enumerate(groups):
        seg = t[j * w:(j + 1) * w]
        cols = range(12, w - 12, 24)[:20]
        alt = []
        for shift in (1, 2):
            x = bytearray(seg)
            for i in cols:
                x[i] = ACGT[(ACGT.index(x[i]) + shift) % 4]
            alt.append(bytes(x))
        for _ in range(n_a):
            s.read(rng, c, j * w, (j + 1) * w, q_a * w, seg=alt[0])
        for _ in range(n_b):
            s.read(rng, c, j * w, (j + 1) * w, None if q_b is None else q_b * w, seg=alt[1])
    # window 4: ordinary reads, so that the set also has a window the weights do not decide
    for _ in range(4):
        s.read(rng, c, 4 * w, 5 * w, _good(rng, w))
    return s


def limits_set(seed: int = 1) -> OverlapSet:
    """The POA batch's limits reached from the cut: a contig of 101 windows (from window 4 on) at depth about 6, one
    window (7) with more than max_sequences_per_poa (200) layers, and one layer longer than max_sequence_size (1023)
    from a read with 1100 bases inserted in the middle of window 12."""
    rng = np.random.default_rng(seed)
    w = 500
    s = OverlapSet(w, first_window=4)
    n = 100 * w + 123
    c = s.contig(_contig(rng, n), _good(rng, n))
    for tb in range(0, n - 200, 150):
        te = min(n, tb + int(rng.integers(600, 1400)))
        s.read(rng, c, tb, te, _good(rng, te - tb) if rng.random() < 0.7 else None)
    for _ in range(205):
        tb = 7 * w + 20 + int(rng.integers(0, 300))
        s.read(rng, c, tb, tb + 120, _good(rng, 120) if rng.random() < 0.7 else None, tag="deep")
    seg = _subst(rng, s.contigs[c][12 * w - 100:13 * w + 100])
    seg = seg[:350] + _contig(rng, 1100) + seg[350:]
    s.read(rng, c, 12 * w - 100, 13 * w + 100, _good(rng, len(seg)), seg=seg, tag="long", gapped=True)
    return s
