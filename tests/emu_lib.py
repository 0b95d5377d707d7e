"""ctypes loader of the host-flavour engine build (tests/emu/libpoa_emu.so; TEST INFRASTRUCTURE)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import _flat_args, _p

HERE = os.path.dirname(os.path.abspath(__file__))

#: per-window reach counters of the emulated fill (enum Reach in tests/emu/emu_poa.cpp), in order
REACH_FIELDS = ("wide1", "wide2", "wide3", "wide4", "chunked_full", "fullw", "chunked_banded", "cells32",
                "general_rows", "far_preds", "jump_preds", "max_npred", "rows_over32", "dyn_rows", "dyn_builds",
                "retries", "retries_full", "max_len")
#: per-window reach counters of the emulated traceback (enum TbReach in tests/emu/emu_poa.cpp), in order
TB_REACH_FIELDS = ("tracebacks", "tile_loads", "reanchors", "global_npred", "global_pred_cap", "global_far",
                   "common_steps", "tile_steps", "neg_chunk_steps", "band_hits", "row0_tail32", "row0_tail64", "vrun32",
                   "count_mod0", "count_mod1", "count_mod31", "i32_reads", "partial_reads", "twin_mismatches")
#: the first traceback of a window that differs from the scalar twin (read -1: none), in order
TB_MISMATCH_FIELDS = ("read", "try", "entry", "twin_node", "twin_pos", "node", "pos", "twin_count", "count")
#: per-window reach counters of the emulated graph phases (enum GraphReach in tests/emu/emu_poa.cpp), in order
GRAPH_REACH_FIELDS = ("new_nodes32", "new_nodes64", "run_cross32", "join1", "join2", "join3", "join4", "join5", "join6",
                      "join7", "clique_mate", "edge_bumped", "edge_created", "edge_same_root", "edge_cross_root",
                      "du_all", "walk_over32", "read_len1", "const_weights", "base_weights", "weight0", "dirty_over32",
                      "sub_serial", "sweep_iter2", "sweep_iter3", "straddle", "straddle8", "sub_begin0",
                      "sub_end_last", "tie_in_block", "tie_pre_block", "tie_equal_pred", "block_max_tie",
                      "max_tie_across", "topsort_twins", "sub_twins", "cons_twins", "twin_mismatches")
#: the first graph twin check of a window that found a difference (kind -1: none; 0 sort, 1 subgraph, 2 consensus)
GRAPH_MISMATCH_FIELDS = ("kind", "read", "index", "twin", "engine")


class Emu:
    def __init__(self):
        subprocess.run(["make", "-s", "-C", os.path.join(HERE, "emu")], check=True,
                       stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(HERE, "emu", "libpoa_emu.so"))

    def polish(self, b, order, m, x, g, max_nodes=4096, max_edges=24576, max_len=1023, band=0,
               serial_topsort=False, threads=8, stride=4096, msa_cap=0, ring_rows=8):
        """Untrimmed consensus, coverage, status and DP cell count of the emulated engine.  Also kept: per sequence
        (ADD order index of the window's first sequence + processing position) the fill digest and fill count
        (last_digest, last_fill_count), per window the reach counters (last_reach: dict REACH_FIELDS -> array).
        ring_rows: the GPU launch's score-row ring, which decides the row program's far-predecessor flags.
        Also per sequence the digest and entry count of the alignment added to the graph (last_aln_digest,
        last_aln_count), per window the traceback's reach counters (last_tb_reach: dict TB_REACH_FIELDS -> array) and
        its first difference from the scalar twin walk (last_tb_mismatch: W x TB_MISMATCH_FIELDS, read -1: none).
        And the graph phases' outputs (last_graph: dict of per-sequence graph_digest, graph_nodes, graph_edges,
        sub_digest, sub_count, per-window cons_digest (W x 2) and cons_rounds), their reach counters (last_graph_reach:
        dict GRAPH_REACH_FIELDS -> array) and first twin difference (last_graph_mismatch: W x GRAPH_MISMATCH_FIELDS)."""
        W = b.n_windows
        cons = np.zeros((W, stride), dtype=np.uint8)
        cov = np.zeros((W, stride), dtype=np.uint16)
        clen = np.zeros(W, dtype=np.int32)
        st = np.zeros(W, dtype=np.int32)
        cells = C.c_int64(0)
        self.last_trim = np.zeros(W, dtype=np.int32)  # device-side trim interval: first | last << 16
        self.last_digest = np.zeros(b.n_seqs, dtype=np.uint64)
        self.last_fill_count = np.zeros(b.n_seqs, dtype=np.int32)
        reach = np.zeros((W, len(REACH_FIELDS)), dtype=np.int32)
        self.last_aln_digest = np.zeros(b.n_seqs, dtype=np.uint64)
        self.last_aln_count = np.zeros(b.n_seqs, dtype=np.int32)
        tb_reach = np.zeros((W, len(TB_REACH_FIELDS)), dtype=np.int32)
        self.last_tb_mismatch = np.full((W, len(TB_MISMATCH_FIELDS)), -1, dtype=np.int32)
        n = b.n_seqs
        gr = {"graph_digest": np.zeros(n, dtype=np.uint64), "graph_nodes": np.zeros(n, dtype=np.int32),
              "graph_edges": np.zeros(n, dtype=np.int32), "sub_digest": np.zeros(n, dtype=np.uint64),
              "sub_count": np.zeros(n, dtype=np.int32), "cons_digest": np.zeros((W, 2), dtype=np.uint64),
              "cons_rounds": np.zeros(W, dtype=np.int32)}
        g_reach = np.zeros((W, len(GRAPH_REACH_FIELDS)), dtype=np.int32)
        self.last_graph_mismatch = np.full((W, len(GRAPH_MISMATCH_FIELDS)), -1, dtype=np.int32)
        order = np.ascontiguousarray(order, dtype=np.int32)
        a = _flat_args(b)
        self.lib.emu_polish_windows_graph(
            a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], _p(order, C.c_int32), C.c_int32(m), C.c_int32(x), C.c_int32(g),
            C.c_int32(max_nodes), C.c_int32(max_edges), C.c_int32(max_len), C.c_int32(band),
            C.c_int32(int(serial_topsort)), C.c_int32(threads), _p(cons, C.c_uint8), _p(cov, C.c_uint16),
            C.c_int32(stride), _p(clen, C.c_int32), _p(st, C.c_int32), None, None, C.byref(cells),
            _p(self.last_trim, C.c_int32), *self._msa_args(W, msa_cap), C.c_int32(ring_rows),
            _p(self.last_digest, C.c_uint64), _p(self.last_fill_count, C.c_int32), _p(reach, C.c_int32),
            _p(self.last_aln_digest, C.c_uint64), _p(self.last_aln_count, C.c_int32), _p(tb_reach, C.c_int32),
            _p(self.last_tb_mismatch, C.c_int32), _p(gr["graph_digest"], C.c_uint64), _p(gr["graph_nodes"], C.c_int32),
            _p(gr["graph_edges"], C.c_int32), _p(gr["sub_digest"], C.c_uint64), _p(gr["sub_count"], C.c_int32),
            _p(gr["cons_digest"], C.c_uint64), _p(gr["cons_rounds"], C.c_int32), _p(g_reach, C.c_int32),
            _p(self.last_graph_mismatch, C.c_int32))
        self.last_graph = gr
        self.last_graph_reach = {k: g_reach[:, i].copy() for i, k in enumerate(GRAPH_REACH_FIELDS)}
        self.last_reach = {k: reach[:, i].copy() for i, k in enumerate(REACH_FIELDS)}
        self.last_tb_reach = {k: tb_reach[:, i].copy() for i, k in enumerate(TB_REACH_FIELDS)}
        self.last_msa = None
        if msa_cap:  # per window: list of rows (processing order), or the status when the MSA failed
            arena, off, cols, mst = self._msa
            nseq = np.diff(b.win_seq_off)
            self.last_msa = [[arena[off[w] + k * cols[w]:off[w] + (k + 1) * cols[w]].tobytes() for k in range(int(nseq[w]))]
                             if mst[w] == 0 else int(mst[w]) for w in range(W)]
        return ([cons[w, :clen[w]].tobytes() for w in range(W)], [cov[w, :clen[w]].copy() for w in range(W)],
                st, cells.value)

    def _msa_args(self, W, msa_cap):
        if not msa_cap:
            self._msa = None
            return (None, C.c_int64(0), None, None, None)
        self._msa = (np.zeros(msa_cap, dtype=np.uint8), np.zeros(W, dtype=np.int64), np.zeros(W, dtype=np.int32),
                     np.zeros(W, dtype=np.int32))
        a, o, c, s = self._msa
        return (_p(a, C.c_uint8), C.c_int64(msa_cap), _p(o, C.c_int64), _p(c, C.c_int32), _p(s, C.c_int32))


class EmuAligner:
    """Host-flavour build of the overlap aligner (tests/emu/libaln_emu.so)."""

    def __init__(self):
        subprocess.run(["make", "-s", "-C", os.path.join(HERE, "emu")], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(HERE, "emu", "libaln_emu.so"))
        self.lib.emu_align.restype = C.c_int64

    def align(self, q: bytes, t: bytes, q_first: int = 0, t_begin: int = 0, window_length: int = 0, guess: int = -1):
        """(ops, edit distance, recursion depth, leaves); self.cigar = the CIGAR formed from the engine's runs"""
        ops = np.zeros(len(q) + len(t) + 8, dtype=np.uint8)
        score, levels, leaves = C.c_int32(-1), C.c_int32(0), C.c_int32(0)
        cap = 4 * (len(q) + len(t)) + 16
        cigar = C.create_string_buffer(cap)
        bp = np.zeros(4 * (len(t) // max(window_length, 1) + 3), dtype=np.uint32)
        bp_count = C.c_int32(0)
        n = self.lib.emu_align(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), _p(ops, C.c_uint8),
                               C.byref(score), C.byref(levels), C.byref(leaves), cigar, C.c_int64(cap),
                               C.c_int32(q_first), C.c_int32(t_begin), C.c_int32(window_length), _p(bp, C.c_uint32),
                               C.byref(bp_count), C.c_int32(guess), C.c_int32(0), None, C.c_int64(0), None, None,
                               C.c_int64(0), None)
        self.breaking_points = bp[:2 * bp_count.value].reshape(-1, 2).copy()  # (t, q) pairs, window_length > 0 only
        assert n >= 0, {-1: "inconsistent split", -2: "list overflow", -3: "runs do not spell the operations"}.get(n, n)
        self.cigar = cigar.value
        return ops[:n].copy(), int(score.value), int(levels.value), int(leaves.value)

    def align_log(self, q: bytes, t: bytes, guess: int = -1, aln: int = 0) -> np.ndarray:
        """The split records (racon_gpu_b200.aligner.SPLIT_REC_DTYPE, path one warp) of aligning one pair as alignment
        `aln` of a batch, every level and every attempt."""
        from racon_gpu_b200.aligner import SPLIT_REC_DTYPE
        assert self.lib.emu_split_rec_bytes() == SPLIT_REC_DTYPE.itemsize
        cap = 4 * (len(q) * len(t) // (1 << 20) + 4) + 64
        log = np.zeros(cap, dtype=SPLIT_REC_DTYPE)
        count = C.c_int64(0)
        ops = np.zeros(len(q) + len(t) + 8, dtype=np.uint8)
        score = C.c_int32(-1)
        n = self.lib.emu_align(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), _p(ops, C.c_uint8),
                               C.byref(score), None, None, None, C.c_int64(0), C.c_int32(0), C.c_int32(0), C.c_int32(0),
                               None, None, C.c_int32(guess), C.c_int32(aln), log.ctypes.data_as(C.c_void_p),
                               C.c_int64(cap), C.byref(count), None, C.c_int64(0), None)
        assert n >= 0 and count.value <= cap, (n, count.value, cap)
        return log[:count.value].copy()

    def align_leaves(self, q: bytes, t: bytes, guess: int = -1, aln: int = 0):
        """The leaf records (racon_gpu_b200.aligner.LEAF_REC_DTYPE) of aligning one pair as alignment `aln` of a batch,
        in the order the leaf list holds them, and the edit distance."""
        from racon_gpu_b200.aligner import LEAF_REC_DTYPE
        assert self.lib.emu_leaf_rec_bytes() == LEAF_REC_DTYPE.itemsize
        cap = 2 * (len(q) * len(t) // (1 << 19) + len(q) + len(t)) // 64 + 64
        log = np.zeros(cap, dtype=LEAF_REC_DTYPE)
        count = C.c_int64(0)
        ops = np.zeros(len(q) + len(t) + 8, dtype=np.uint8)
        score = C.c_int32(-1)
        n = self.lib.emu_align(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), _p(ops, C.c_uint8),
                               C.byref(score), None, None, None, C.c_int64(0), C.c_int32(0), C.c_int32(0), C.c_int32(0),
                               None, None, C.c_int32(guess), C.c_int32(aln), None, C.c_int64(0), None,
                               log.ctypes.data_as(C.c_void_p), C.c_int64(cap), C.byref(count))
        assert n >= 0 and count.value <= cap, (n, count.value, cap)
        return log[:count.value].copy(), int(score.value)

    #: emu_leaf's slot contents before the pass: zeros, 0xFF, 0xA5, seeded random bytes, another leaf's leftovers
    POISONS = ("zero", "ff", "a5", "random", "leftovers")

    def leaf(self, q: bytes, t: bytes, band: int, poison: str = "zero", seed: int = 0, other=None):
        """One leaf the way aln_leaf_kernel runs it, in a slot filled per `poison` first (other = (q, t, band) of the leaf
        whose leftovers the slot holds).  Returns (the (n + m)-byte operations region, the LEAF_REC_DTYPE record)."""
        from racon_gpu_b200.aligner import LEAF_REC_DTYPE
        self.lib.emu_leaf.restype = C.c_int64
        region = np.zeros(len(q) + len(t) + 1, dtype=np.uint8)
        rec = np.zeros(1, dtype=LEAF_REC_DTYPE)
        pq, pt, pband = other if other is not None else (b"", b"", -1)
        self.lib.emu_leaf(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), C.c_int32(band),
                          C.c_int32(self.POISONS.index(poison)), C.c_uint64(seed), C.c_char_p(pq), C.c_int32(len(pq)),
                          C.c_char_p(pt), C.c_int32(len(pt)), C.c_int32(pband), _p(region, C.c_uint8),
                          rec.ctypes.data_as(C.c_void_p))
        return region[:len(q) + len(t)].copy(), rec[0]

    def ops_digest(self, region: np.ndarray) -> int:
        """aln_ops_digest of an operations region (holes 0xFF included)."""
        self.lib.emu_ops_digest.restype = C.c_uint64
        region = np.ascontiguousarray(region, dtype=np.uint8)
        return int(self.lib.emu_ops_digest(_p(region, C.c_uint8), C.c_int32(region.shape[0])))

    #: emu_split's stats, in order
    SPLIT_STATS = ("stripes", "left_matrix", "anchors", "other", "waits", "failures", "timeouts")

    def split(self, q: bytes, t: bytes, best: int = -1, guess: bool = False, team: bool = False, seed: int = 0):
        """One Hirschberg step of the sub-problem (q, t) the way a split kernel runs it: one warp, or (team=True) a team
        block on 2 x ALN_TEAM threads under the protocol checker.  best < 0: no band; guess: best is the host's guess
        (redone without a band when the optimum is larger).  Returns a list of attempts, each a dict with Lc, Rr (n + 1
        values), r, ls, rs, best, band; team mode also self.last_stats (SPLIT_STATS) and self.last_failure."""
        n, m = len(q), len(t)
        Lc = np.zeros(2 * (n + 1), dtype=np.int32)
        Rr = np.zeros(2 * (n + 1), dtype=np.int32)
        sp = np.zeros(8, dtype=np.int32)
        band = np.zeros(2, dtype=np.int32)
        stats = np.zeros(7, dtype=np.int64)
        msg = C.create_string_buffer(512)
        self.lib.emu_split.restype = C.c_int32
        k = self.lib.emu_split(C.c_char_p(q), C.c_int32(n), C.c_char_p(t), C.c_int32(m), C.c_int32(best),
                               C.c_int32(int(guess)), C.c_int32(int(team)), C.c_uint64(seed), _p(Lc, C.c_int32),
                               _p(Rr, C.c_int32), _p(sp, C.c_int32), _p(band, C.c_int32), _p(stats, C.c_int64), msg,
                               C.c_int32(512))
        self.last_stats = dict(zip(self.SPLIT_STATS, stats.tolist()))
        self.last_failure = msg.value.decode()
        return [{"Lc": Lc[a * (n + 1):(a + 1) * (n + 1)].copy(), "Rr": Rr[a * (n + 1):(a + 1) * (n + 1)].copy(),
                 "r": int(sp[4 * a]), "ls": int(sp[4 * a + 1]), "rs": int(sp[4 * a + 2]), "best": int(sp[4 * a + 3]),
                 "band": int(band[a])} for a in range(k)]
