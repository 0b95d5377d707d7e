"""CPU: racon's window-layer cut (racon_gpu_b200/csrc/layer_cut.cuh) in its host build (tests/emu/emu_cut.cpp),
against the windows the unmodified racon built from the lambda-phage sample and against a plain restatement of
src/polisher.cpp:403-457 on generated breaking points; and the ctypes mirrors of the cut's structs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from common import lambda_fixture, overlap_fixture
from cut_cases import racon_layers

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LAYER = np.dtype([("q_off", "<i8"), ("window", "<i4"), ("length", "<i4"), ("begin", "<i4"), ("end", "<i4"),
                  ("has_quality", "<i4"), ("overlap", "<i4")])


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_cut") / "libcut_emu.so"
    subprocess.run(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-x", "c++", "-o", str(so),
                    os.path.join(HERE, "emu", "emu_cut.cpp")], check=True)
    lib = C.CDLL(str(so))
    lib.emu_layer_cut.restype = C.c_int64
    lib.emu_cut_scan.restype = None
    assert lib.emu_cut_layer_bytes() == LAYER.itemsize
    return lib


def _p(a, ty):
    return a.ctypes.data_as(C.POINTER(ty))


def run_cut(lib, ov, w, threshold, n_win, win_lo=0, seed=1):
    """ov: list of dicts {q (bytes, the read segment), qual (bytes or None), q_first, bp ((k, 2) uint32 (t, q)),
    first_window}.  Returns (records, counts)."""
    q_arena = b"".join(o["q"] for o in ov)
    qual_arena = b"".join(o["qual"] if o["qual"] is not None else b"\0" * len(o["q"]) for o in ov)
    q_off = np.concatenate([[0], np.cumsum([len(o["q"]) for o in ov])[:-1]]).astype(np.int64)
    bp_count = np.asarray([o["bp"].shape[0] for o in ov], dtype=np.int32)
    bp_off = np.concatenate([[0], np.cumsum(bp_count)[:-1]]).astype(np.int64)
    bp = np.ascontiguousarray(np.concatenate([o["bp"].reshape(-1) for o in ov] + [np.zeros(4, np.uint32)]), dtype=np.uint32)
    fw = np.asarray([o["first_window"] for o in ov], dtype=np.int64)
    qf = np.asarray([o["q_first"] for o in ov], dtype=np.int32)
    hq = np.asarray([o["qual"] is not None for o in ov], dtype=np.uint8)
    qual = np.frombuffer(qual_arena + b"\0", dtype=np.uint8).copy()
    out = np.zeros(max(int(bp_count.sum()) // 2, 1), dtype=LAYER)
    counts = np.zeros(max(n_win, 1), dtype=np.int32)
    kept = lib.emu_layer_cut(C.c_int32(len(ov)), _p(q_off, C.c_int64), _p(bp_off, C.c_int64), _p(bp_count, C.c_int32),
                             _p(fw, C.c_int64), _p(qf, C.c_int32), _p(hq, C.c_uint8), _p(bp, C.c_uint32),
                             _p(qual, C.c_uint8), C.c_int32(w), C.c_double(threshold), C.c_int64(win_lo),
                             C.c_int64(n_win), C.c_uint64(seed), out.ctypes.data_as(C.c_void_p), _p(counts, C.c_int32))
    return out[:kept], counts[:n_win], q_arena, qual_arena


def lambda_overlaps(case):
    """racon's filtered overlap list of a lambda run (tests/golden/make_layer_golden.py) with the real breaking points."""
    z = np.load(os.path.join(HERE, "golden", "lambda_layers.npz"))
    ovf = overlap_fixture()
    qual, hq = z[f"{case}_qual"].tobytes(), z[f"{case}_has_q"]
    out, pos = [], 0
    for i, src in enumerate(z[f"{case}_src"]):
        o = ovf[int(src)]
        q = None
        if hq[i]:
            q = qual[pos:pos + len(o["q"])]
            pos += len(o["q"])
        out.append({"q": o["q"], "qual": q, "q_first": o["q_first"], "t_begin": o["t_begin"], "t": o["t"],
                    "bp": o["bp"].astype(np.uint32), "first_window": 0, "strand": int(z[f"{case}_strand"][i])})
    return out


@pytest.mark.parametrize("case", ["fastq_500", "fasta_500"])
@pytest.mark.parametrize("seed", [1, 2])
def test_cut_reproduces_racon_lambda_windows(emu, case, seed):
    """Every layer of every window -- bytes, weights, begin, end, add order, per-window count -- equals the window
    racon built (tests/golden/lambda_windows.npz), whatever order the scatter ran in."""
    b, _, _, p = lambda_fixture(case)
    ov = lambda_overlaps(case)
    assert any(o["strand"] for o in ov) and any(not o["strand"] for o in ov)
    rec, counts, q_arena, qual_arena = run_cut(emu, ov, p["window_length"], 10.0, b.n_windows, seed=seed)
    nseq = np.diff(b.win_seq_off)
    assert (counts == nseq - 1).all()
    assert (np.diff(rec["window"]) >= 0).all()
    k = 0
    for w in range(b.n_windows):
        for s in range(int(b.win_seq_off[w]) + 1, int(b.win_seq_off[w + 1])):
            r = rec[k]
            k += 1
            assert r["window"] == w
            lo, hi = int(r["q_off"]), int(r["q_off"] + r["length"])
            assert q_arena[lo:hi] == b.bases[b.seq_off[s]:b.seq_off[s + 1]].tobytes(), (w, s)
            assert (int(r["begin"]), int(r["end"])) == (int(b.begins[s]), int(b.ends[s]))
            assert bool(r["has_quality"]) == bool(b.has_weights[s])
            if r["has_quality"]:
                wts = (np.frombuffer(qual_arena[lo:hi], dtype=np.uint8).astype(np.int16) - 33).astype(np.int8)
                assert (wts == b.weights[b.seq_off[s]:b.seq_off[s + 1]]).all()
    assert k == rec.shape[0]
    if case == "fastq_500":  # the quality filter dropped layers here, and not for the FASTA reads
        assert rec.shape[0] < run_cut(emu, ov, 500, -1.0, b.n_windows)[0].shape[0]


def synth_overlaps(rng, w, threshold):
    """Overlaps on three contigs with breaking points racon could form: each touches consecutive windows of its contig
    and covers each with one aligned stretch.  Planted edges: a layer of exactly 0.02 * w bases, one just below; a mean
    quality exactly at the threshold, one just below; reads without qualities; an overlap keeping no layer; the short
    last window of a contig; a one-column window (begin == end)."""
    contigs = [(0, 1730), (4, 1400), (8, 999)]  # (first window, length)
    ov = []
    for k in range(60):
        ci = int(rng.integers(len(contigs)))
        fw, tl = contigs[ci]
        nwin = (tl + w - 1) // w
        a = int(rng.integers(nwin))
        bnd = int(rng.integers(a, nwin)) + 1
        pts, q, qlen = [], int(rng.integers(0, 50)), []
        q_first = q
        for win in range(a, bnd):
            lo, hi = win * w, min((win + 1) * w, tl)
            t0 = int(rng.integers(lo, hi))
            t1 = int(rng.integers(t0 + 1, hi + 1))
            ln = int(rng.integers(1, 2 * (t1 - t0) + 2))
            kind = k % 9
            if kind == 1:
                ln = int(round(0.02 * w))  # exactly 0.02 * w: kept
            elif kind == 2:
                ln = int(round(0.02 * w)) - 1  # just below: dropped
            elif kind == 7 and win == a:
                t1 = t0 + 1  # one aligned column: begin == end
            pts += [(t0, q), (t1, q + ln)]
            qlen.append(ln)
            q += ln + int(rng.integers(0, 5))
        n = q - q_first
        seq = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=n).tobytes()
        kind = k % 9
        if kind == 3:
            qual = None  # FASTA read
        else:
            qual = bytearray(rng.integers(33 + 2, 33 + 40, size=n, dtype=np.uint8).tobytes())
            if kind in (4, 5):  # a mean exactly at the threshold (kept), and one quality point below it (dropped)
                for (t0, q0), (t1, q1) in zip(pts[0::2], pts[1::2]):
                    for i in range(q0 - q_first, q1 - q_first):
                        qual[i] = 33 + int(threshold)
                    if kind == 5:
                        qual[q0 - q_first] -= 1
            elif kind == 6:  # every layer below the threshold: the overlap keeps nothing
                qual = bytearray(b"\x23" * n)
            qual = bytes(qual)
        ov.append({"q": seq, "qual": qual, "q_first": q_first, "bp": np.asarray(pts, dtype=np.uint32).reshape(-1, 2),
                   "first_window": fw})
    return ov, 10  # windows 0 .. 9 (id 7 unused)


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_cut_matches_racon_restatement(emu, seed):
    w, thr = 500, 10.0
    rng = np.random.default_rng(seed)
    ov, n_win = synth_overlaps(rng, w, thr)
    want = racon_layers(ov, [o["bp"] for o in ov], w, thr)
    rec, counts, _, _ = run_cut(emu, ov, w, thr, n_win, seed=seed)
    got = {}
    q_off = np.concatenate([[0], np.cumsum([len(o["q"]) for o in ov])[:-1]])
    for r in rec:
        k = int(r["overlap"])
        q0 = int(r["q_off"] - q_off[k]) + ov[k]["q_first"]
        got.setdefault(int(r["window"]), []).append((k, q0, int(r["length"]), int(r["begin"]), int(r["end"]),
                                                     bool(r["has_quality"])))
    assert got == want
    assert [counts[x] for x in range(n_win)] == [len(want.get(x, [])) for x in range(n_win)]
    # the planted edges were reached
    lens = [x[2] for v in want.values() for x in v]
    assert 10 in lens and 9 not in lens
    kept = {x[0] for v in want.values() for x in v}
    assert any(k % 9 == 6 for k in range(len(ov)) if k not in kept)  # overlaps that keep no layer
    assert any(k % 9 == 4 for k in kept) and not any(k % 9 == 5 for k in kept)  # mean == threshold kept, below dropped
    assert any(not x[5] for v in want.values() for x in v)  # reads without qualities
    # the short last windows of contigs 1 and 3 (230 and 499 bases)
    assert 3 in want and max(x[4] for x in want[3]) < 230 and 9 in want and max(x[4] for x in want[9]) < 499


@pytest.mark.parametrize("n_win", [0, 1, 1023, 1024, 1025, 2049, 10000])
def test_cut_scan_matches_cumsum(emu, n_win):
    """Phase 2 (aln_cut_scan_kernel's body, run for its 1024 threads): every window's offset is the exclusive prefix
    sum of the counts, and win_off[n_win] their total, also where a thread owns more than one window (n_win > 1024)
    and where the last threads own none."""
    rng = np.random.default_rng(n_win)
    counts = rng.integers(0, 300, size=max(n_win, 1)).astype(np.int32)[:n_win]
    counts[rng.random(n_win) < 0.3] = 0  # empty windows between kept ones
    win_off = np.full(n_win + 1, -7, dtype=np.int64)
    emu.emu_cut_scan(_p(np.ascontiguousarray(counts), C.c_int32), C.c_int64(n_win), _p(win_off, C.c_int64))
    want = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)])
    assert (win_off == want).all(), int(np.flatnonzero(win_off != want)[0])


@pytest.mark.parametrize("header,name,fields", [("b200aln.h", "b200aln_layer", ["overlap", "window", "begin"]),
                                                ("b200aln.h", "b200aln_layer_inputs", ["has_quality", "q_quality"]),
                                                ("b200poa.h", "b200poa_overlap_options",
                                                 ["aligner_mem", "quality_threshold", "max_windows_per_batch"])])
def test_cut_struct_layouts(tmp_path, header, name, fields):
    from racon_gpu_b200.aligner import AlnLayer, AlnLayerInputs
    from racon_gpu_b200.api import OverlapOptions
    cls = {"b200aln_layer": AlnLayer, "b200aln_layer_inputs": AlnLayerInputs, "b200poa_overlap_options": OverlapOptions}[name]
    src = tmp_path / "sz.c"
    body = 'printf("%%zu\\n", sizeof(%s));' % name + "".join('printf("%%zu\\n", offsetof(%s, %s));' % (name, f)
                                                                for f in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){%s return 0;}\n' % (header, body))
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(cls)] + [getattr(cls, f).offset for f in fields]
    if name == "b200aln_layer":
        assert C.sizeof(cls) == LAYER.itemsize
