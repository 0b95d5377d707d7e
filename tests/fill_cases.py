"""The DP fill at its edges: window sets, the emulation's reach report for each, and a runner for the GPU side.

Every case is a list of runs (one batch configuration over one window set).  The CPU suite runs each run through the
emulation (tests/emu: ScalarFill, the scalar twin of poa_fill.cuh) and asserts the run reaches the fill path its name
promises (tests/test_fill_reach.py); the GPU suite runs the same batches on the device and compares per-read fill
digests, status, consensus, coverage and MSA rows with the emulation (tests/test_gpu_fill.py).

`python fill_cases.py IN OUT` is the GPU worker: it runs the jobs pickled in IN on the library named by B200POA_LIB
(api.load_library() loads one library per process, so the digest build runs in a process of its own) and pickles the
results to OUT.
"""
from __future__ import annotations

import ctypes as C
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from racon_gpu_b200.windows import WindowBatch, synth_windows  # noqa: E402

M, X, G = 3, -5, -4
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
GB = 1 << 30


def run(name, batch, mode="full", band=256, msz=1023, scoring=(M, X, G), env=None, depth=200, mem=2 * GB):
    """One batch: mode full / static / adaptive, band = static width or the adaptive band's first try (exact: not
    rounded to 128 the way b200poa_config_default rounds it), msz = max_sequence_size, depth = max_sequences_per_poa."""
    return {"name": name, "batch": batch, "mode": mode, "band": band, "msz": msz, "scoring": tuple(scoring),
            "env": dict(env or {}), "depth": depth, "mem": mem}


def max_nodes(r):
    """b200poa_config_default: 3 x max_sequence_size nodes in full band, 4 x when banded."""
    return ((3 if r["mode"] == "full" else 4) * r["msz"] + 3) // 4 * 4


# ------------------------------------------------------------------------------------------------------------------
# window builders
# ------------------------------------------------------------------------------------------------------------------
def _fit(seq: bytes, wt, n: int, rng):
    """seq (and its weights) cut or padded with random bases to exactly n bases."""
    s = seq[:n] + rng.choice(ACGT, size=max(0, n - len(seq))).tobytes()
    if wt is not None:
        wt = np.concatenate([wt[:n], np.zeros(max(0, n - len(wt)), dtype=np.int8)])
    return s, wt


def _window(seqs, wts, spans=None):
    L = len(seqs[0])
    out = [(seqs[0], wts[0], 0, 0)]
    for i in range(1, len(seqs)):
        bg, en = spans[i] if spans else (0, L - 1)
        out.append((seqs[i], wts[i], bg, en))
    return out


#: read lengths whose colsP = (len + 1 + 7) & ~7 falls on both sides of 256, 512, 768 and 1024 columns
LADDER = (247, 248, 255, 256, 263, 504, 511, 512, 760, 767, 768, 1016, 1023, 1024, 1100)


def ladder_windows(depth: int = 5) -> WindowBatch:
    """One window per ladder length: backbone and every read exactly that long."""
    rng = np.random.default_rng(11)
    wins = []
    for T in LADDER:
        seqs, wts, _, _ = synth_windows(1, T, depth, 0.1, seed=T).window(0)
        fitted = [_fit(s, w, T, rng) for s, w in zip(seqs, wts)]
        wins.append(_window([f[0] for f in fitted], [f[1] for f in fitted]))
    return WindowBatch.from_lists(wins)


def colsp(n: int) -> int:
    return (n + 1 + 7) & ~7


def big_graph_windows() -> WindowBatch:
    """Reads (longer than the widest band) against a much longer backbone: the graph has about twice as many rows as
    the read has columns, and more with every read."""
    rng = np.random.default_rng(12)
    wins = []
    for w in range(3):
        seqs, wts, _, _ = synth_windows(1, 940, 6, 0.1, seed=120 + w).window(0)
        reads = []
        for s in seqs[1:]:
            a = int(rng.integers(0, len(s) - 540))
            reads.append(s[a:a + 530])
        wins.append(_window([seqs[0]] + reads, [wts[0]] + [None] * len(reads)))
    return WindowBatch.from_lists(wins)


def long_read_windows() -> WindowBatch:
    """Reads several times longer than the backbone: the band start moves by several columns per row, more than the
    ring rows' back pad over a few rows."""
    wins = []
    for w in range(3):
        seqs, wts, _, _ = synth_windows(1, 700, 8, 0.1, seed=130 + w).window(0)
        bb, bw = seqs[0][320:380], wts[0][320:380]
        wins.append(_window([bb] + seqs[1:], [bw] + wts[1:]))
    return WindowBatch.from_lists(wins)


def mixed_length_windows() -> WindowBatch:
    """One window per set: reads shorter than any band (fill_rows_wide) next to reads longer than the widest."""
    lens = (30, 50, 60, 90, 120, 200, 260, 300, 400, 500, 560, 10 ** 6)
    wins = []
    for w in range(2):
        seqs, wts, _, _ = synth_windows(1, 600, len(lens), 0.1, seed=140 + w).window(0)
        reads = [s[:n] for s, n in zip(seqs[1:], lens)]
        wins.append(_window([seqs[0]] + reads, [wts[0]] + [None] * len(reads)))
    return WindowBatch.from_lists(wins)


def concat(*batches: WindowBatch) -> WindowBatch:
    wins = []
    for b in batches:
        for w in range(b.n_windows):
            wins.append(list(zip(*b.window(w))))
    return WindowBatch.from_lists(wins)


IUPAC = np.frombuffer(b"NRYKMSWBDHVNNacgtn", dtype=np.uint8)


def odd_letter_windows() -> WindowBatch:
    """Backbones and reads with N, IUPAC codes and lowercase letters, scattered and in alternating runs (every letter
    change in a run of graph rows rebuilds the fill's on-demand profile row)."""
    rng = np.random.default_rng(13)
    b = synth_windows(6, 300, 10, 0.1, seed=150)
    wins = []
    for w in range(b.n_windows):
        seqs, wts, bg, en = b.window(w)
        out = []
        for s, wt in zip(seqs, wts):
            a = np.frombuffer(s, dtype=np.uint8).copy()
            hit = rng.random(a.shape[0]) < 0.03
            a[hit] = rng.choice(IUPAC, size=int(hit.sum()))
            k = int(rng.integers(20, a.shape[0] - 40))
            a[k:k + 16] = np.frombuffer(b"NRNRNRYKYKacacNN", dtype=np.uint8)
            out.append(a.tobytes())
        wins.append(list(zip(out, wts, bg, en)))
    return WindowBatch.from_lists(wins)


def ladder_of_lengths(n: int = 200, lo: int = 60, hi: int = 1100, depth: int = 5) -> WindowBatch:
    """n windows from lo to hi bases (slot reuse: the longest-first work list hands a slot windows of falling size)."""
    wins = []
    for w in range(n):
        L = lo + (hi - lo) * w // (n - 1)
        wins.append(list(zip(*synth_windows(1, L, depth, 0.1, seed=1000 + w).window(0))))
    return WindowBatch.from_lists(wins)


def deep_windows() -> WindowBatch:
    """200 reads at 28 % error; 150 reads that either lack a stretch of 1-139 bases ending at one backbone position or
    carry a random insertion of 1-11 bases just before it, so that the position's node gets more than 32
    predecessors; and two of cudapoa's deep sample windows."""
    from common import cudapoa_fixture
    rng = np.random.default_rng(1)
    truth = rng.choice(ACGT, 300).tobytes()
    reads = []
    for i in range(150):
        k = int(rng.integers(1, 140))
        if i % 2:
            reads.append(truth[:150 - k] + truth[150:])
        else:
            reads.append(truth[:150] + rng.choice(ACGT, int(rng.integers(1, 12))).tobytes() + truth[150:])
    hub = WindowBatch.from_lists([_window([truth] + reads, [None] * 151)])
    cb, _, _ = cudapoa_fixture()
    return concat(synth_windows(1, 250, 200, 0.28, seed=160), hub, cb.slice(0, 2))


def short_deletion_windows() -> WindowBatch:
    """Every other read lacks 100-140 consecutive bases of a 320-base window: from a narrow first band the adaptive
    retries double the width until the full matrix."""
    rng = np.random.default_rng(17)
    wins = []
    for w in range(3):
        seqs, wts, _, _ = synth_windows(1, 320, 10, 0.08, seed=170 + w).window(0)
        reads = []
        for i, s in enumerate(seqs[1:]):
            if i % 2:
                a, d = int(rng.integers(60, 120)), int(rng.integers(100, 140))
                s = s[:a] + s[a + d:]
            reads.append(s)
        wins.append(_window([seqs[0]] + reads, wts))
    return WindowBatch.from_lists(wins)


# ------------------------------------------------------------------------------------------------------------------
# the cases: name -> list of runs
# ------------------------------------------------------------------------------------------------------------------
BAND_WIDTHS = (256, 64, 128, 200, 384, 512)
SCORINGS = ((10, -10, -60), (60, -60, -60), (40, -30, -50), (2, 1, -1), (0, -1, -1), (127, -1, 0))
SWITCHING = SCORINGS[:3]  # int16 cells for the first reads of a window, 32-bit cells once the graph has grown


def band_sets():
    """(name, batch) of the window sets every static band width runs over."""
    from common import partial_span_windows
    return [("big_graph", big_graph_windows()), ("long_reads", long_read_windows()),
            ("mixed", mixed_length_windows()), ("partial", partial_span_windows(n=4))]


def cases():
    from test_emu import deletion_windows
    small = synth_windows(6, 300, 10, 0.12, seed=21)
    out = {}
    out["ladder"] = [run("ladder", ladder_windows(), msz=1279)]
    out["ring"] = [run("ring8", small, msz=2047),
                   run("ring2", concat(small, synth_windows(1, 1330, 4, 0.04, seed=22)), msz=2047),
                   run("ring16", synth_windows(8, 70, 12, 0.1, seed=23)),
                   run("ring32", synth_windows(8, 20, 12, 0.1, seed=24)),
                   run("ring_bytes1", synth_windows(8, 500, 32, 0.15, seed=25), env={"B200POA_RING_BYTES": 1}),
                   run("ring_bytes1_static", synth_windows(8, 500, 32, 0.15, seed=25), mode="static",
                       env={"B200POA_RING_BYTES": 1})]
    bands = concat(*[b for _, b in band_sets()])
    out["bands"] = [run(f"static{w}", bands, mode="static", band=w) for w in BAND_WIDTHS]
    adapt = concat(deletion_windows(n=4), short_deletion_windows(), synth_windows(4, 500, 16, 0.12, seed=26))
    out["adaptive"] = [run(f"adaptive{w}", adapt, mode="adaptive", band=w) for w in (64, 128)]
    deep = deep_windows()
    out["deep"] = [run("deep_full", deep, msz=2047, depth=256), run("deep_static", deep, mode="static", msz=2047, depth=256)]
    odd = odd_letter_windows()
    out["letters"] = [run("letters_full", odd), run("letters_static256", odd, mode="static"),
                      run("letters_static128", odd, mode="static", band=128),
                      run("letters_adaptive128", odd, mode="adaptive", band=128)]
    sc_runs = []
    for sc in SCORINGS:
        # switching scorings: windows just around the read length at which int16 stops being provably enough
        L = {SWITCHING[0]: 450, SWITCHING[1]: 262, SWITCHING[2]: 350}.get(sc, 200)
        b = synth_windows(3, L, 16, 0.15, seed=27)
        tag = "%d_%d_%d" % sc
        sc_runs += [run(f"scoring{tag}_full", b, scoring=sc),
                    run(f"scoring{tag}_static256", b, mode="static", scoring=sc),
                    run(f"scoring{tag}_static128", b, mode="static", band=128, scoring=sc),
                    run(f"scoring{tag}_adaptive128", b, mode="adaptive", band=128, scoring=sc)]
    out["scoring"] = sc_runs
    reuse = ladder_of_lengths()
    slot = []
    for mode in ("full", "static"):
        slot.append(run(f"reuse_clean_{mode}", reuse, mode=mode, msz=1279, mem=4 * GB))
        for poison in (165, 60):
            slot.append(run(f"reuse_poison{poison}_{mode}", reuse, mode=mode, msz=1279, mem=4 * GB,
                            env={"B200POA_SLAB_FILL": poison, "B200POA_BLOCKS_PER_SM": 1}))
    out["slot_reuse"] = slot
    return out


# ------------------------------------------------------------------------------------------------------------------
# the emulation side
# ------------------------------------------------------------------------------------------------------------------
def msa_capacity(b: WindowBatch, msz: int) -> int:
    nseq = np.diff(b.win_seq_off)
    tot = np.add.reduceat(np.diff(b.seq_off), b.win_seq_off[:-1])
    return int((nseq * np.minimum(tot, 2 * msz) + 16).sum()) + 64


def emu_run(emu, r, ring_rows: int, msa: bool = True):
    """The run through the emulation at the GPU launch's ring size: dict of status, consensus, coverage, MSA (or
    None), per-sequence digests and fill counts (processing order), per-window reach counters."""
    from racon_gpu_b200 import api
    b = r["batch"]
    m, x, g = r["scoring"]
    band = {"full": 0, "static": r["band"], "adaptive": -r["band"]}[r["mode"]]
    cons, cov, st, _ = emu.polish(b, api.processing_order(b), m, x, g, max_nodes=max_nodes(r), max_len=r["msz"],
                                  band=band, stride=2 * r["msz"], msa_cap=msa_capacity(b, r["msz"]) if msa else 0,
                                  ring_rows=ring_rows)
    return {"status": st, "cons": cons, "cov": cov, "msa": emu.last_msa, "digest": emu.last_digest.copy(),
            "count": emu.last_fill_count.copy(), "reach": emu.last_reach, "aln_digest": emu.last_aln_digest.copy(),
            "aln_count": emu.last_aln_count.copy(), "tb_reach": emu.last_tb_reach,
            "tb_mismatch": emu.last_tb_mismatch.copy(), "trim": emu.last_trim.copy(),
            "graph": {k: v.copy() for k, v in emu.last_graph.items()}, "graph_reach": emu.last_graph_reach,
            "graph_mismatch": emu.last_graph_mismatch.copy()}


def ring_rows_of(r) -> int:
    """The ring smem_geometry() (b200poa.cu) gives a launch whose longest staged read is that of the run's batch."""
    b = r["batch"]
    c = colsp(int(np.diff(b.seq_off).max()))
    banded = r["mode"] == "static" and r["band"] < c
    row = (max(r["band"], 256) if banded else c) + 8 + 24
    ring_bytes = 4096
    if 4096 < 16 * row <= 20480:
        ring_bytes = 16 * row
    if "B200POA_RING_BYTES" in r["env"]:
        ring_bytes = int(r["env"]["B200POA_RING_BYTES"])
    rows = 2
    while rows < 32 and rows * 4 * row <= ring_bytes:
        rows *= 2
    return rows


def reach_failures(name: str, rep: dict, b: WindowBatch, r) -> list:
    """What the run `name` must reach, from the emulation's report; returns the unmet promises."""
    tot = {k: int(v.sum()) for k, v in rep.items()}
    need = []
    if name == "ladder":
        want = {"wide1": 3, "wide2": 4, "wide3": 3, "wide4": 3, "chunked_full": 2}
        for w, T in enumerate(LADDER):
            c = colsp(T)
            v = "wide1" if c <= 256 else "wide2" if c <= 512 else "wide3" if c <= 768 else "wide4" if c <= 1024 else "chunked_full"
            n = int(np.diff(b.win_seq_off)[w]) - 1
            if rep[v][w] != n:
                need.append(f"window {w} (length {T}): {n} reads through {v}, got {rep[v][w]}")
        for v, k in want.items():
            if int((rep[v] > 0).sum()) != k:
                need.append(f"{k} windows through {v}")
    elif name.startswith("ring"):
        want = {"ring8": 8, "ring2": 2, "ring16": 16, "ring32": 32, "ring_bytes1": 2, "ring_bytes1_static": 2}[name]
        if ring_rows_of(r) != want:
            need.append(f"a {want}-row ring (host rule gives {ring_rows_of(r)})")
        if want == 2 and (tot["far_preds"] == 0 or tot["general_rows"] == 0):
            need.append("predecessors outside a 2-row ring")
    elif name.startswith("static"):
        w = int(name[len("static"):])
        banded = "fullw" if w == 256 else "chunked_banded"
        sets = [n for n, _ in band_sets()]
        sizes = [bb.n_windows for _, bb in band_sets()]
        lo = dict(zip(sets, np.cumsum([0] + sizes[:-1])))
        hi = dict(zip(sets, np.cumsum(sizes)))
        sl = lambda s, k: rep[k][lo[s]:hi[s]]
        longest = np.maximum.reduceat(np.diff(b.seq_off), b.win_seq_off[:-1])
        for s in sets:  # every window with a read longer than the band
            if not ((sl(s, banded) > 0) | (np.asarray([colsp(int(n)) for n in longest[lo[s]:hi[s]]]) <= w)).all():
                need.append(f"{s}: every window banded through {banded}")
        if sl("big_graph", banded).sum() == 0 or sl("long_reads", banded).sum() == 0:
            need.append("big_graph and long_reads banded")
        if not ((sl("mixed", "wide1") > 0) & (sl("mixed", banded) > 0)).all():
            need.append("mixed: reads shorter and longer than the band in one window")
        if w < 512 and sl("long_reads", "jump_preds").sum() == 0:
            need.append("long_reads: band starts jumping more than RING_PAD_BACK")
        other = "chunked_banded" if w == 256 else "fullw"
        if tot[other]:
            need.append(f"no read through {other}")
    elif name.startswith("adaptive"):
        if tot["retries"] == 0 or tot["retries_full"] == 0:
            need.append("adaptive retries up to the full matrix")
    elif name.startswith("deep"):
        if tot["rows_over32"] == 0 or tot["far_preds"] == 0 or tot["general_rows"] == 0:
            need.append("rows with more than 32 predecessors and predecessors outside the ring")
    elif name.startswith("letters"):
        if (rep["dyn_rows"] == 0).any() or tot["dyn_builds"] < 100:
            need.append("the on-demand profile row in every window, rebuilt often")
    elif name.startswith("scoring"):
        sc = r["scoring"]
        if sc in SWITCHING and not ((rep["cells32"] > 0) & (rep["cells32"] < np.diff(b.win_seq_off) - 1)).any():
            need.append("int16 and 32-bit cells inside one window")
        if sc not in SWITCHING and tot["cells32"]:
            need.append("int16 cells only")
    elif name.startswith("reuse"):
        L = np.diff(b.seq_off)[b.win_seq_off[:-1]]
        if L.min() > 80 or L.max() < 1050:
            need.append("windows from 60 to 1100 bases")
    return need


# ------------------------------------------------------------------------------------------------------------------
# the GPU side
# ------------------------------------------------------------------------------------------------------------------
def gpu_runs(runs, digest: bool = True):
    """Run the batches in a process of their own on the digest build (or the product library).  Returns one dict per
    run: status, cons, cov, msa, ring_rows, ring_stride and, on the digest build, digest and count."""
    from racon_gpu_b200 import build
    lib = build.DIGEST_LIB if digest else build.LIB
    if not os.path.exists(lib):
        raise RuntimeError(f"{lib} is missing: run __graft_entry__.build()")
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.pkl"), os.path.join(d, "out.pkl")
        with open(src, "wb") as fh:
            pickle.dump([dict(r, digest=digest) for r in runs], fh)
        env = dict(os.environ, B200POA_LIB=lib)
        subprocess.run([sys.executable, os.path.abspath(__file__), src, dst], env=env, check=True, cwd=ROOT)
        with open(dst, "rb") as fh:
            return pickle.load(fh)


def _gpu_job(r):
    from racon_gpu_b200 import api

    class ExactBatch(api.PoaBatch):
        """A batch created from an explicit configuration (the band width as given)."""

        def __init__(self, cfg, r):
            self.lib = api.load_library(build_if_missing=False)
            self.cfg = cfg
            self.handle = C.c_void_p()
            m, x, g = r["scoring"]
            st = self.lib.b200poa_batch_create(C.c_int32(0), C.c_void_p(0), C.c_size_t(r["mem"]),
                                               C.c_int32(api.OUTPUT_CONSENSUS | api.OUTPUT_MSA), C.byref(cfg),
                                               C.c_int16(g), C.c_int16(x), C.c_int16(m), C.byref(self.handle))
            if st != api.SUCCESS:
                raise RuntimeError(f"b200poa_batch_create failed: {api.status_string(st)}")

    old = {k: os.environ.get(k) for k in r["env"]}
    os.environ.update({k: str(v) for k, v in r["env"].items()})
    try:
        lib = api.load_library(build_if_missing=False)
        cfg = api.Config()
        mode = {"full": api.FULL_BAND, "static": api.STATIC_BAND, "adaptive": api.ADAPTIVE_BAND}[r["mode"]]
        lib.b200poa_config_default(C.byref(cfg), C.c_int32(r["msz"]), C.c_int32(r["depth"]), C.c_int32(r["band"]),
                                   C.c_int32(mode))
        cfg.alignment_band_width = r["band"]
        pb = ExactBatch(cfg, r)
        b = r["batch"]
        n, added = pb.add_windows(b)
        assert n == b.n_windows and (np.asarray(added) == np.diff(b.win_seq_off) - 1).all(), "the batch dropped input"
        pb.generate_poa()
        cons, cov, status = pb.get_consensus()
        msa, msa_status = pb.get_msa()
        out = {"status": status, "cons": cons, "cov": cov, "msa": msa, "msa_status": msa_status}
        if r["digest"]:
            dg = np.zeros(b.n_seqs, dtype=np.uint64)
            cnt = np.zeros(b.n_seqs, dtype=np.int32)
            rr, rs = C.c_int32(0), C.c_int32(0)
            st = lib.b200poa_debug_fill_digest(pb.handle, dg.ctypes.data_as(C.POINTER(C.c_uint64)),
                                               cnt.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(b.n_seqs),
                                               C.byref(rr), C.byref(rs))
            assert st == api.SUCCESS, api.status_string(st)
            out.update(digest=dg, count=cnt, ring_rows=rr.value, ring_stride=rs.value)
            adg = np.zeros(b.n_seqs, dtype=np.uint64)
            acnt = np.zeros(b.n_seqs, dtype=np.int32)
            st = lib.b200poa_debug_aln_digest(pb.handle, adg.ctypes.data_as(C.POINTER(C.c_uint64)),
                                              acnt.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(b.n_seqs))
            assert st == api.SUCCESS, api.status_string(st)
            out.update(aln_digest=adg, aln_count=acnt)
            n, W = b.n_seqs, b.n_windows
            gr = {"graph_digest": np.zeros(n, dtype=np.uint64), "graph_nodes": np.zeros(n, dtype=np.int32),
                  "graph_edges": np.zeros(n, dtype=np.int32), "sub_digest": np.zeros(n, dtype=np.uint64),
                  "sub_count": np.zeros(n, dtype=np.int32), "cons_digest": np.zeros((W, 2), dtype=np.uint64),
                  "cons_rounds": np.zeros(W, dtype=np.int32)}
            ptr = {k: v.ctypes.data_as(C.POINTER(C.c_uint64 if v.dtype == np.uint64 else C.c_int32))
                   for k, v in gr.items()}
            st = lib.b200poa_debug_graph_digest(pb.handle, ptr["graph_digest"], ptr["graph_nodes"], ptr["graph_edges"],
                                                ptr["sub_digest"], ptr["sub_count"], C.c_int64(n), ptr["cons_digest"],
                                                ptr["cons_rounds"], C.c_int64(W))
            assert st == api.SUCCESS, api.status_string(st)
            out.update(graph=gr)
        pb.close()
        return out
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def aln_digest_failures(name, b, got, want, what="emulation") -> list:
    """Per window, the first read (processing position) whose alignment digest or entry count differs."""
    bad = []
    for w in range(b.n_windows):
        s0, s1 = int(b.win_seq_off[w]), int(b.win_seq_off[w + 1])
        for k in range(s1 - s0):
            s = s0 + k
            if got["aln_count"][s] != want["aln_count"][s] or got["aln_digest"][s] != want["aln_digest"][s]:
                bad.append(f"{name}: window {w} read {k}: alignment of {got['aln_count'][s]} entries digest "
                           f"{got['aln_digest'][s]:#x}, {what} {want['aln_count'][s]} entries digest "
                           f"{want['aln_digest'][s]:#x}")
                break
    return bad


SEQ_FIELDS = ("graph_digest", "graph_nodes", "graph_edges", "sub_digest", "sub_count")


def graph_digest_failures(name, b, got, want, what="emulation", windows=None) -> list:
    """Per window (all, or those listed), the first read (processing position) whose graph or subgraph digest or count
    differs, and a differing consensus digest or round count."""
    bad = []
    for w in (range(b.n_windows) if windows is None else windows):
        s0, s1 = int(b.win_seq_off[w]), int(b.win_seq_off[w + 1])
        for k in range(s1 - s0):
            diff = [f for f in SEQ_FIELDS if got[f][s0 + k] != want[f][s0 + k]]
            if diff:
                bad.append(f"{name}: window {w} read {k}: {', '.join(diff)} differ from the {what} ("
                           f"{got['graph_nodes'][s0 + k]} nodes {got['graph_edges'][s0 + k]} edges, {what} "
                           f"{want['graph_nodes'][s0 + k]} nodes {want['graph_edges'][s0 + k]} edges)")
                break
        for j, when in enumerate(("after the scoring pass", "after branch completion")):
            if got["cons_digest"][w][j] != want["cons_digest"][w][j]:
                bad.append(f"{name}: window {w}: consensus scores {when} differ from the {what}")
        if got["cons_rounds"][w] != want["cons_rounds"][w]:
            bad.append(f"{name}: window {w}: {got['cons_rounds'][w]} rounds of branch completion, {what} "
                       f"{want['cons_rounds'][w]}")
    return bad



def compare(r, got, want, oracle_out=None) -> list:
    """Differences between a GPU run and the emulation (and, in full band, the oracle).  Digest mismatches name the
    window, the read (processing position) and how many fills it took; alignment digests (where both sides have them)
    the read and its entry counts; graph digests the read and its node and edge counts."""
    b = r["batch"]
    bad = []
    if "aln_digest" in got and "aln_digest" in want:
        bad += aln_digest_failures(r["name"], b, got, want)
    if "graph" in got and "graph" in want:
        bad += graph_digest_failures(r["name"], b, got["graph"], want["graph"])
    if "digest" in got:
        for w in range(b.n_windows):
            s0, s1 = int(b.win_seq_off[w]), int(b.win_seq_off[w + 1])
            for k in range(s1 - s0):
                s = s0 + k
                if got["count"][s] != want["count"][s] or got["digest"][s] != want["digest"][s]:
                    bad.append(f"{r['name']}: window {w} read {k}: {got['count'][s]} fills digest {got['digest'][s]:#x}, "
                               f"emulation {want['count'][s]} fills digest {want['digest'][s]:#x}")
                    break
    for w in range(b.n_windows):
        if got["status"][w] != want["status"][w]:
            bad.append(f"{r['name']}: window {w} status {got['status'][w]} != {want['status'][w]}")
        elif got["cons"][w] != want["cons"][w] or not np.array_equal(got["cov"][w], want["cov"][w]):
            bad.append(f"{r['name']}: window {w} consensus/coverage differs from the emulation")
        elif want["msa"] is not None and got["msa"][w] != (want["msa"][w] if not isinstance(want["msa"][w], int) else None):
            bad.append(f"{r['name']}: window {w} MSA differs from the emulation")
    if oracle_out is not None:
        oc, ocov, omsa = oracle_out
        for w in range(b.n_windows):
            if got["cons"][w] != oc[w] or not np.array_equal(got["cov"][w], ocov[w]):
                bad.append(f"{r['name']}: window {w} consensus/coverage differs from the oracle")
            elif omsa is not None and got["msa"][w] is None:  # racon_gpu's limit: max_consensus_size columns or more
                if not (got["msa_status"][w] == 2 and len(omsa[w][0]) >= 2 * r["msz"]):
                    bad.append(f"{r['name']}: window {w} has no MSA (status {got['msa_status'][w]})")
            elif omsa is not None and got["msa"][w] != omsa[w]:
                bad.append(f"{r['name']}: window {w} MSA differs from the oracle")
    return bad


def oracle_outputs(oracle, r, msa: bool = True):
    """Full band: the oracle's untrimmed consensus, coverage and (optionally) MSA rows of the run's windows."""
    from oracle_lib import oracle_window_msa, window_sequences
    from racon_gpu_b200 import api
    b = r["batch"]
    m, x, g = r["scoring"]
    order = api.processing_order(b)
    oc, ocov, _ = oracle.polish(b, order, m, x, g, tgs=False, trim=False, threads=16, stride=8192)
    omsa = None
    if msa:
        omsa = []
        for w in range(b.n_windows):
            seqs, wts, bg, en = window_sequences(b, order, w)
            omsa.append(oracle_window_msa(oracle, seqs, wts, bg, en, m, x, g))
    return oc, ocov, omsa


if __name__ == "__main__":
    with open(sys.argv[1], "rb") as fh:
        jobs = pickle.load(fh)
    results = [_gpu_job(r) for r in jobs]
    with open(sys.argv[2], "wb") as fh:
        pickle.dump(results, fh)
