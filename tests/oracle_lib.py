"""ctypes loaders for the parity checkers (TEST INFRASTRUCTURE: tests/, smoke(), bench cpu legs only).

  Oracle  -> oracle/liboracle.so          plain-C restatement of racon's spoa path
  Ref     -> oracle/_ref/libracon_ref.so  the unmodified reference (racon::Window + spoa), built
                                          from the reference's sources by oracle/Makefile
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")


def build_oracle(quiet: bool = True) -> None:
    """(Re)build liboracle.so and, when the reference's sources are present, _ref/libracon_ref.so."""
    subprocess.run(["make", "-s", "-C", ORACLE_DIR], check=True,
                   stdout=subprocess.DEVNULL if quiet else None,
                   stderr=subprocess.DEVNULL if quiet else None)


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


def _flat_args(b):
    return (C.c_int64(b.n_windows), _p(b.win_seq_off, C.c_int64), _p(b.seq_off, C.c_int64),
            _p(b.bases, C.c_uint8), _p(b.weights, C.c_int8), _p(b.has_weights, C.c_uint8),
            _p(b.begins, C.c_int32), _p(b.ends, C.c_int32))


class Oracle:
    def __init__(self):
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            build_oracle()
        self.lib = C.CDLL(path)
        self.lib.poa_oracle_polish_windows.restype = None

    def polish(self, batch, order: np.ndarray, m: int, x: int, g: int, tgs: bool = True,
               trim: bool = True, threads: int = 1, stride: int = 4096, want_stats: bool = False):
        """Returns (list of consensus bytes, list of coverage arrays, polished flags[, stats])."""
        W = batch.n_windows
        cons = np.zeros((W, stride), dtype=np.uint8)
        cov = np.zeros((W, stride), dtype=np.uint16)
        clen = np.zeros(W, dtype=np.int32)
        pol = np.zeros(W, dtype=np.uint8)
        stats = np.zeros((W, 6), dtype=np.int64)
        order = np.ascontiguousarray(order, dtype=np.int32)
        self.lib.poa_oracle_polish_windows(
            *_flat_args(batch), _p(order, C.c_int32), C.c_int32(int(tgs)), C.c_int32(int(trim)),
            C.c_int32(m), C.c_int32(x), C.c_int32(g), C.c_int32(threads),
            cons.ctypes.data_as(C.c_char_p), _p(cov, C.c_uint16), C.c_int32(stride),
            _p(clen, C.c_int32), _p(pol, C.c_uint8), _p(stats, C.c_int64))
        assert (clen >= 0).all(), "oracle output stride too small"
        out = [cons[w, :clen[w]].tobytes() for w in range(W)]
        covs = [cov[w, :clen[w]].copy() for w in range(W)]
        if want_stats:
            return out, covs, pol.astype(bool), stats
        return out, covs, pol.astype(bool)

    def alignment_digests(self, batch, order: np.ndarray, m: int, x: int, g: int, threads: int = 16):
        """Per sequence (ADD-order index of the window's first sequence + processing position): the digest and pair
        count of the alignment spoa adds to the window's graph (poa_oracle_alignment_digests; 0, 0 for backbones)."""
        dg = np.zeros(batch.n_seqs, dtype=np.uint64)
        cnt = np.zeros(batch.n_seqs, dtype=np.int32)
        order = np.ascontiguousarray(order, dtype=np.int32)
        self.lib.poa_oracle_alignment_digests.restype = None
        self.lib.poa_oracle_alignment_digests(*_flat_args(batch), _p(order, C.c_int32), C.c_int32(m), C.c_int32(x),
                                              C.c_int32(g), C.c_int32(threads), _p(dg, C.c_uint64),
                                              _p(cnt, C.c_int32))
        return dg, cnt

    def graph_digests(self, batch, order: np.ndarray, m: int, x: int, g: int, threads: int = 16) -> dict:
        """spoa's graphs hashed the way the engine's test build hashes its own (poa_oracle_graph_digests): per sequence
        (ADD-order index of the window's first sequence + processing position) graph_digest, graph_nodes, graph_edges,
        sub_digest and sub_count; per window cons_digest (W x 2), cons_rounds, overflow (weights or scores that do
        not fit 32 bits) and max_indegree (the largest in-degree of the final graph)."""
        n, W = batch.n_seqs, batch.n_windows
        out = {"graph_digest": np.zeros(n, dtype=np.uint64), "graph_nodes": np.zeros(n, dtype=np.int32),
               "graph_edges": np.zeros(n, dtype=np.int32), "sub_digest": np.zeros(n, dtype=np.uint64),
               "sub_count": np.zeros(n, dtype=np.int32), "cons_digest": np.zeros((W, 2), dtype=np.uint64),
               "cons_rounds": np.zeros(W, dtype=np.int32), "overflow": np.zeros(W, dtype=np.int64),
               "max_indegree": np.zeros(W, dtype=np.int32)}
        order = np.ascontiguousarray(order, dtype=np.int32)
        self.lib.poa_oracle_graph_digests.restype = None
        self.lib.poa_oracle_graph_digests(
            *_flat_args(batch), _p(order, C.c_int32), C.c_int32(m), C.c_int32(x), C.c_int32(g), C.c_int32(threads),
            _p(out["graph_digest"], C.c_uint64), _p(out["graph_nodes"], C.c_int32), _p(out["graph_edges"], C.c_int32),
            _p(out["sub_digest"], C.c_uint64), _p(out["sub_count"], C.c_int32), _p(out["cons_digest"], C.c_uint64),
            _p(out["cons_rounds"], C.c_int32), _p(out["overflow"], C.c_int64), _p(out["max_indegree"], C.c_int32))
        return out


def _seq_arrays(seqs, weights):
    n = len(seqs)
    arr_s = (C.c_char_p * n)(*[bytes(s) for s in seqs])
    lens = np.asarray([len(s) for s in seqs], dtype=np.int32)
    keep = [None if w is None else np.ascontiguousarray(w, dtype=np.int8) for w in weights]
    arr_w = (C.POINTER(C.c_int8) * n)(*[
        C.cast(None, C.POINTER(C.c_int8)) if w is None else _p(w, C.c_int8) for w in keep])
    return n, arr_s, lens, keep, arr_w


def window_sequences(batch, order: np.ndarray, w: int):
    """Window w of a flat batch as (seqs, weights, begins, ends) in PROCESSING order."""
    s0, s1 = int(batch.win_seq_off[w]), int(batch.win_seq_off[w + 1])
    seqs, wts, bg, en = [], [], [], []
    for k in range(s1 - s0):
        s = s0 + int(order[s0 + k])
        a, b = int(batch.seq_off[s]), int(batch.seq_off[s + 1])
        seqs.append(batch.bases[a:b].tobytes())
        wts.append(batch.weights[a:b].copy() if batch.has_weights[s] else None)
        bg.append(int(batch.begins[s]))
        en.append(int(batch.ends[s]))
    return seqs, wts, bg, en


def oracle_window_msa(oracle: "Oracle", seqs, weights, begins, ends, m: int, x: int, g: int):
    """spoa's MSA (one row per sequence, processing order) of a window built like racon builds it; begins None:
    every layer spans the window (a plain cudapoa group)."""
    lib = oracle.lib
    n, arr_s, lens, keep, arr_w = _seq_arrays(seqs, weights)
    rows = C.c_void_p()
    L = C.c_int32(0)
    lib.poa_oracle_window_msa.restype = C.c_int32
    bg = None if begins is None else np.ascontiguousarray(begins, dtype=np.int32)
    en = None if begins is None else np.ascontiguousarray(ends, dtype=np.int32)
    nr = lib.poa_oracle_window_msa(C.c_int32(n), arr_s, _p(lens, C.c_int32), arr_w,
                                   None if bg is None else _p(bg, C.c_int32),
                                   None if en is None else _p(en, C.c_int32),
                                   C.c_int32(m), C.c_int32(x), C.c_int32(g), C.byref(rows), C.byref(L))
    buf = C.string_at(rows.value, nr * L.value)
    lib.poa_oracle_free.argtypes = [C.c_void_p]
    lib.poa_oracle_free(rows)
    return [buf[i * L.value:(i + 1) * L.value] for i in range(nr)]


class Ref:
    """The unmodified reference.  `available` is False when oracle/_ref was not built."""

    def __init__(self):
        path = os.path.join(ORACLE_DIR, "_ref", "libracon_ref.so")
        if not os.path.exists(path) and os.path.isdir("vendor/spoa/src"):
            build_oracle()
        self.available = os.path.exists(path)
        self.lib = C.CDLL(path) if self.available else None

    def layer_order(self, begins: np.ndarray) -> np.ndarray:
        begins = np.ascontiguousarray(begins, dtype=np.int32)
        out = np.zeros(begins.shape[0], dtype=np.int32)
        self.lib.ref_layer_order(C.c_int32(begins.shape[0]), _p(begins, C.c_int32), _p(out, C.c_int32))
        return out

    def polish(self, batch, m: int, x: int, g: int, tgs: bool = True, trim: bool = True,
               threads: int = 1, window_length: int = 500, stride: int = 4096):
        W = batch.n_windows
        cons = np.zeros((W, stride), dtype=np.uint8)
        clen = np.zeros(W, dtype=np.int32)
        pol = np.zeros(W, dtype=np.uint8)
        self.lib.ref_polish_windows(
            *_flat_args(batch), C.c_int32(int(tgs)), C.c_int32(int(trim)), C.c_int32(m),
            C.c_int32(x), C.c_int32(g), C.c_int32(window_length), C.c_int32(threads),
            cons.ctypes.data_as(C.c_char_p), C.c_int32(stride), _p(clen, C.c_int32),
            _p(pol, C.c_uint8))
        assert (clen <= stride).all()
        return [cons[w, :clen[w]].tobytes() for w in range(W)], pol.astype(bool)

    def spoa_window(self, seqs, weights, m: int, x: int, g: int, max_nodes: int = 1 << 16):
        """seqs in PROCESSING order.  Returns (consensus, coverage, rank_to_node)."""
        n = len(seqs)
        arr_s = (C.c_char_p * n)(*[bytes(s) for s in seqs])
        lens = np.asarray([len(s) for s in seqs], dtype=np.int32)
        keep = [None if w is None else np.ascontiguousarray(w, dtype=np.int8) for w in weights]
        arr_w = (C.POINTER(C.c_int8) * n)(*[
            C.cast(None, C.POINTER(C.c_int8)) if w is None else _p(w, C.c_int8) for w in keep])
        max_out = int(lens.sum()) + 8
        cons = np.zeros(max_out, dtype=np.uint8)
        cov = np.zeros(max_out, dtype=np.uint32)
        rank = np.zeros(max_nodes, dtype=np.int32)
        nn = C.c_int32(0)
        self.lib.ref_spoa_window.restype = C.c_int32
        ln = self.lib.ref_spoa_window(
            C.c_int32(n), arr_s, _p(lens, C.c_int32), arr_w, C.c_int32(m), C.c_int32(x),
            C.c_int32(g), cons.ctypes.data_as(C.c_char_p), _p(cov, C.c_uint32), C.c_int32(max_out),
            _p(rank, C.c_int32), C.c_int32(max_nodes), C.byref(nn))
        return cons[:ln].tobytes(), cov[:ln].copy(), rank[:nn.value].copy()


def ref_window_msa(ref: Ref, seqs, weights, m: int, x: int, g: int):
    """spoa::Graph::generate_multiple_sequence_alignment of the unmodified reference for one group."""
    n, arr_s, lens, keep, arr_w = _seq_arrays(seqs, weights)
    cap = int(lens.sum()) * n + 64
    out = np.zeros(cap, dtype=np.uint8)
    L = C.c_int32(0)
    ref.lib.ref_spoa_window_msa.restype = C.c_int32
    nr = ref.lib.ref_spoa_window_msa(C.c_int32(n), arr_s, _p(lens, C.c_int32), arr_w, C.c_int32(m), C.c_int32(x),
                                     C.c_int32(g), out.ctypes.data_as(C.c_char_p), C.c_int64(cap), C.byref(L))
    assert nr * L.value <= cap
    return [out[i * L.value:(i + 1) * L.value].tobytes() for i in range(nr)]


def processing_order(batch, layer_order_fn) -> np.ndarray:
    """order[s] for a flat batch using a layer-order function (begins[n] -> rank[n])."""
    order = np.zeros(batch.n_seqs, dtype=np.int32)
    for w in range(batch.n_windows):
        s0, s1 = int(batch.win_seq_off[w]), int(batch.win_seq_off[w + 1])
        order[s0:s1] = layer_order_fn(batch.begins[s0:s1])
    return order


# ---------------------------------------------------------------------------------------------------
# overlap alignment (edlib NW path): oracle/aln_oracle.c restatement and the unmodified edlib in oracle/_ref
# ---------------------------------------------------------------------------------------------------
def oracle_align(oracle: "Oracle", q: bytes, t: bytes):
    """(ops uint8 array, edit distance) of the restatement; ops: 0 match, 1 insertion, 2 deletion, 3 mismatch."""
    cap = len(q) + len(t) + 8
    ops = np.zeros(cap, dtype=np.uint8)
    score = C.c_int32(0)
    oracle.lib.aln_oracle_nw.restype = C.c_int64
    n = oracle.lib.aln_oracle_nw(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), _p(ops, C.c_uint8),
                                 C.c_int64(cap), C.byref(score))
    assert n >= 0
    return ops[:n].copy(), int(score.value)


def oracle_last_column(oracle: "Oracle", q: bytes, t: bytes) -> np.ndarray:
    """col[i] = D[i][len(t)] of the plain edit-distance matrix of q against t, i = 0..len(q)."""
    col = np.zeros(len(q) + 1, dtype=np.int32)
    oracle.lib.aln_oracle_last_column.restype = None
    oracle.lib.aln_oracle_last_column(C.c_char_p(q), C.c_int32(len(q)), C.c_int(1), C.c_char_p(t), C.c_int32(len(t)),
                                      C.c_int(1), _p(col, C.c_int32))
    return col


def ops_to_cigar(oracle: "Oracle", ops: np.ndarray) -> bytes:
    ops = np.ascontiguousarray(ops, dtype=np.uint8)
    cap = 16 * ops.shape[0] + 16
    buf = C.create_string_buffer(cap)
    oracle.lib.aln_oracle_cigar.restype = C.c_int64
    n = oracle.lib.aln_oracle_cigar(_p(ops, C.c_uint8), C.c_int64(ops.shape[0]), buf, C.c_int64(cap))
    assert n >= 0
    return buf.raw[:n]


def ref_align(ref: "Ref", q: bytes, t: bytes):
    """(ops, edit distance, CIGAR) of the unmodified edlib called like racon calls it (src/overlap.cpp:205-224)."""
    cap = len(q) + len(t) + 8
    ops = np.zeros(cap, dtype=np.uint8)
    ccap = 16 * cap
    cig = C.create_string_buffer(ccap)
    score = C.c_int32(0)
    ref.lib.ref_edlib_nw.restype = C.c_int64
    n = ref.lib.ref_edlib_nw(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), _p(ops, C.c_uint8),
                             C.c_int64(cap), cig, C.c_int64(ccap), C.byref(score))
    assert n >= 0
    return ops[:n].copy(), int(score.value), cig.value


def oracle_breaking_points(oracle: "Oracle", ops: np.ndarray, q_first: int, t_begin: int, t_end: int, window_length: int):
    """(t, q) pairs, two per window with a match (restatement of src/overlap.cpp:226-290 on operations)."""
    ops = np.ascontiguousarray(ops, dtype=np.uint8)
    cap = 2 * ((t_end - t_begin) // window_length + 3)
    out = np.zeros(2 * cap, dtype=np.uint32)
    oracle.lib.aln_oracle_breaking_points.restype = C.c_int64
    n = oracle.lib.aln_oracle_breaking_points(_p(ops, C.c_uint8), C.c_int64(ops.shape[0]), C.c_int32(q_first),
                                              C.c_int32(t_begin), C.c_int32(t_end), C.c_int32(window_length),
                                              _p(out, C.c_uint32), C.c_int64(cap))
    assert n >= 0
    return out[:2 * n].reshape(-1, 2).copy()


def ref_breaking_points(ref: "Ref", cigar: bytes, q_length: int, q_begin: int, q_end: int, strand: int, t_length: int,
                        t_begin: int, t_end: int, window_length: int):
    """The unmodified racon::Overlap::find_breaking_points (src/overlap.cpp:179-203,226-290) fed this CIGAR."""
    cap = 2 * ((t_end - t_begin) // window_length + 3)
    out = np.zeros(2 * cap, dtype=np.uint32)
    ref.lib.ref_racon_breaking_points.restype = C.c_int64
    n = ref.lib.ref_racon_breaking_points(C.c_char_p(cigar), C.c_uint32(q_length), C.c_uint32(q_begin), C.c_uint32(q_end),
                                          C.c_int(strand), C.c_uint32(t_length), C.c_uint32(t_begin), C.c_uint32(t_end),
                                          C.c_uint32(window_length), _p(out, C.c_uint32), C.c_int64(cap))
    assert n >= 0
    return out[:2 * n].reshape(-1, 2).copy()
