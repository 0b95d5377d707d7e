"""ctypes binding of the overlap aligner's C ABI (include/b200aln.h) -- for tests and bench.py only.

Mirrors racon's adapter for this step, racon::CUDABatchAligner (src/cuda/cudaaligner.hpp:24-96:
addOverlap / alignAll / generate_cigar_strings / reset) one level below racon's Overlap objects: a pair is
(query = read segment, target = contig segment) exactly as Overlap::align_overlaps hands them to edlib
(src/overlap.cpp:205-209).  The product is the CUDA library; there is no CPU fallback here."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .api import load_library

#: every symbol include/b200aln.h declares (tests check the library exports all of them)
ALN_ABI_SYMBOLS = (
    "b200aln_init", "b200aln_batch_create", "b200aln_batch_add_alignment", "b200aln_batch_align_all",
    "b200aln_batch_sync", "b200aln_batch_num_alignments", "b200aln_batch_get_alignment", "b200aln_batch_get_cigar",
    "b200aln_batch_get_ops", "b200aln_batch_reset", "b200aln_batch_destroy", "b200aln_batch_get_info",
    "b200aln_status_string", "b200aln_align_pairs", "b200aln_batch_add_alignments", "b200aln_batch_get_cigars",
    "b200aln_aligner_create", "b200aln_aligner_num_batches", "b200aln_aligner_align", "b200aln_aligner_destroy",
    "b200aln_batch_set_window_length", "b200aln_batch_add_overlap", "b200aln_batch_add_overlaps",
    "b200aln_batch_get_breaking_points", "b200aln_batch_add_overlaps_view", "b200aln_host_register",
    "b200aln_host_unregister", "b200aln_batch_set_band_guess",
)

SUCCESS, UNINITIALIZED, EXCEEDED_MAX_ALIGNMENTS, EXCEEDED_MAX_LENGTH = 0, 1, 2, 3
GENERIC_ERROR, INVALID_ARGUMENT, CUDA_ERROR = 5, 6, 7


#: one record of the test build's split log (aln_core.cuh AlnSplitRec, b200aln_debug_split_log): a Hirschberg split
#: attempt -- the sub-problem, the band its passes got, attempt 0 or 1 (redone without a band), level, path (SPLIT_PATHS),
#: flags (1: a team_wait gave up), the split and order-independent hashes of both middle columns
SPLIT_REC_DTYPE = np.dtype([("aln", "<i4"), ("r0", "<i4"), ("c0", "<i4"), ("n", "<i4"), ("m", "<i4"), ("band", "<i4"),
                            ("attempt", "<i4"), ("level", "<i4"), ("path", "<i4"), ("flags", "<i4"), ("r", "<i4"),
                            ("ls", "<i4"), ("rs", "<i4"), ("best", "<i4"), ("pad", "<i4", (2,)), ("lc_hash", "<u8"),
                            ("rr_hash", "<u8")])
SPLIT_PATHS = ("warp", "team", "side")  # one warp; a team in a thin level; a team on the side stream
SPLIT_TIMEOUT = 1

#: one record of the test build's leaf log (aln_core.cuh AlnLeafRec, b200aln_debug_leaf_log): a leaf -- the sub-problem,
#: the band its pass got, its flags (bit 0 top level, bit 1 guessed band), the score at its last cell, the walk's counters
#: (LEAF_COUNTERS), the cells its pass computed and an order-independent hash of its (n + m)-byte operations region
LEAF_COUNTERS = ("diag_rounds", "diag_ops", "matches", "up_rounds", "left_rounds", "full_runs", "reload_block",
                 "reload_col", "border_lanes", "tail", "tail_kind")
LEAF_REC_DTYPE = np.dtype([("aln", "<i4"), ("r0", "<i4"), ("c0", "<i4"), ("n", "<i4"), ("m", "<i4"), ("band", "<i4"),
                           ("top", "<i4"), ("score", "<i4")] + [(k, "<i4") for k in LEAF_COUNTERS]
                          + [("pad", "<i4"), ("cells", "<i8"), ("ops_hash", "<u8")])


def is_leaf(n: int, m: int) -> bool:
    """aln_core.cuh aln_is_leaf (edlib.cpp:1135-1157): is an n x m sub-problem traced back without a split?"""
    return n == 0 or m == 0 or 20 * ((n + 63) // 64) * m + 8 * m < 1024 * 1024


class AlnBatchInfo(C.Structure):
    _fields_ = [("device_id", C.c_int32), ("n_slots", C.c_int32), ("levels", C.c_int32), ("kernel_launches", C.c_int32),
                ("team_launches", C.c_int32), ("n_team_blocks", C.c_int32),
                ("n_open", C.c_int64), ("n_leaves", C.c_int64), ("cells", C.c_int64), ("h2d_bytes", C.c_int64),
                ("d2h_bytes", C.c_int64), ("kernel_ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def _lib():
    lib = load_library()
    if not getattr(lib, "_aln_typed", False):
        lib.b200aln_status_string.restype = C.c_char_p
        lib.b200aln_batch_destroy.restype = None
        lib.b200aln_aligner_destroy.restype = None
        lib.b200aln_batch_get_cigar.restype = C.c_int64
        lib.b200aln_batch_get_ops.restype = C.c_int64
        lib._aln_typed = True
    return lib


def status_string(st: int) -> str:
    return _lib().b200aln_status_string(C.c_int32(int(st))).decode()


class CUDABatchAligner:
    """One aligner batch on one device (createCUDABatchAligner(max_bandwidth, device_id, max_gpu_memory),
    src/cuda/cudaaligner.cpp:18-45)."""

    def __init__(self, device_id: int = 0, max_gpu_memory: int = 0, max_bandwidth: int = 0, stream=None):
        self.lib = _lib()
        self.h = C.c_void_p()
        st = self.lib.b200aln_batch_create(C.c_int32(device_id), C.c_void_p(stream), C.c_int64(int(max_gpu_memory)),
                                           C.c_int32(max_bandwidth), C.byref(self.h))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_create: {status_string(st)}")

    def close(self):
        if self.h:
            self.lib.b200aln_batch_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_overlap(self, query: bytes, target: bytes) -> bool:
        """CUDABatchAligner::addOverlap (cudaaligner.cpp:50-81): False = the batch is full (align, reset, add again)."""
        st = self.lib.b200aln_batch_add_alignment(self.h, C.c_char_p(query), C.c_int32(len(query)), C.c_char_p(target),
                                                  C.c_int32(len(target)))
        if st == EXCEEDED_MAX_ALIGNMENTS:
            return False
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_add_alignment: {status_string(st)}")
        return True

    def add_overlaps(self, q: np.ndarray, q_off: np.ndarray, t: np.ndarray, t_off: np.ndarray, first: int = 0,
                     q_first: np.ndarray | None = None, t_begin: np.ndarray | None = None, view: bool = False) -> int:
        """b200aln_batch_add_overlaps[_view] from pair `first` on: how many went in before the batch was full.
        view=True: no staging copy, the arrays must stay alive and unchanged until align_all has returned."""
        n = len(q_off) - 1 - first
        added = C.c_int64(0)
        p = lambda a, ty: a.ctypes.data_as(C.POINTER(ty))
        qf = p(np.ascontiguousarray(q_first[first:], dtype=np.int32), C.c_int32) if q_first is not None else None
        tb = p(np.ascontiguousarray(t_begin[first:], dtype=np.int32), C.c_int32) if t_begin is not None else None
        fn = self.lib.b200aln_batch_add_overlaps_view if view else self.lib.b200aln_batch_add_overlaps
        st = fn(self.h, C.c_int64(n), p(q, C.c_uint8), p(q_off[first:], C.c_int64), p(t, C.c_uint8), p(t_off[first:], C.c_int64),
                qf, tb, C.byref(added))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_add_overlaps: {status_string(st)}")
        return int(added.value)

    def set_band_guess(self, permille: int):
        """-1: learn the top level's band from the previous align_all (default); 0: never band the top level; > 0: fixed."""
        st = self.lib.b200aln_batch_set_band_guess(self.h, C.c_int32(permille))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_set_band_guess: {status_string(st)}")

    def set_window_length(self, window_length: int, skip_cigars: bool = False):
        """Form breaking points on the device (Overlap::find_breaking_points_from_cigar, src/overlap.cpp:226-290)."""
        st = self.lib.b200aln_batch_set_window_length(self.h, C.c_int32(window_length), C.c_int32(1 if skip_cigars else 0))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_set_window_length: {status_string(st)}")

    def breaking_points(self):
        """After align_all: list of (k, 2) uint32 arrays of (t, q), one per overlap (Overlap::breaking_points())."""
        st = self.lib.b200aln_batch_sync(self.h)
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_sync: {status_string(st)}")
        n = self.lib.b200aln_batch_num_alignments(self.h)
        pts, off, cnt = C.POINTER(C.c_uint32)(), C.POINTER(C.c_int64)(), C.POINTER(C.c_int32)()
        st = self.lib.b200aln_batch_get_breaking_points(self.h, C.byref(pts), C.byref(off), C.byref(cnt))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_get_breaking_points: {status_string(st)}")
        if n == 0:
            return []
        off_a = np.ctypeslib.as_array(off, shape=(n,))
        cnt_a = np.ctypeslib.as_array(cnt, shape=(n,))
        total = int((off_a + cnt_a).max())
        flat = np.ctypeslib.as_array(pts, shape=(max(2 * total, 1),))
        return [flat[2 * off_a[k]:2 * (off_a[k] + cnt_a[k])].reshape(-1, 2).copy() for k in range(n)]

    def cigars(self):
        """b200aln_batch_get_cigars after sync: (text bytes view, off int64[n], len int32[n], edit distance int32[n])."""
        st = self.lib.b200aln_batch_sync(self.h)
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_sync: {status_string(st)}")
        n = self.lib.b200aln_batch_num_alignments(self.h)
        text, off, ln, ed, ast = C.c_void_p(), C.POINTER(C.c_int64)(), C.POINTER(C.c_int32)(), C.POINTER(C.c_int32)(), C.POINTER(C.c_int32)()
        st = self.lib.b200aln_batch_get_cigars(self.h, C.byref(text), C.byref(off), C.byref(ln), C.byref(ed), C.byref(ast))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_get_cigars: {status_string(st)}")
        if n == 0:
            return b"", np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32)
        off_a = np.ctypeslib.as_array(off, shape=(n,)).copy()
        len_a = np.ctypeslib.as_array(ln, shape=(n,)).copy()
        ed_a = np.ctypeslib.as_array(ed, shape=(n,)).copy()
        st_a = np.ctypeslib.as_array(ast, shape=(n,))
        if (st_a != SUCCESS).any():
            raise RuntimeError(f"alignment {int(np.flatnonzero(st_a != SUCCESS)[0])}: {status_string(int(st_a[st_a != SUCCESS][0]))}")
        total = int((off_a + len_a).max()) + 1
        return C.string_at(text, total), off_a, len_a, ed_a

    def has_overlaps(self) -> bool:
        return self.lib.b200aln_batch_num_alignments(self.h) > 0

    def align_all(self):
        """CUDABatchAligner::alignAll (cudaaligner.cpp:83-86)"""
        st = self.lib.b200aln_batch_align_all(self.h)
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_align_all: {status_string(st)}")

    def generate_cigar_strings(self):
        """CUDABatchAligner::generate_cigar_strings (cudaaligner.cpp:88-103): list of (cigar bytes, edit distance)."""
        st = self.lib.b200aln_batch_sync(self.h)
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_batch_sync: {status_string(st)}")
        out = []
        for k in range(self.lib.b200aln_batch_num_alignments(self.h)):
            ed, ast = C.c_int32(-1), C.c_int32(-1)
            self.lib.b200aln_batch_get_alignment(self.h, C.c_int32(k), None, None, None, C.byref(ed), C.byref(ast))
            if ast.value != SUCCESS:
                raise RuntimeError(f"alignment {k}: {status_string(ast.value)}")
            n = self.lib.b200aln_batch_get_cigar(self.h, C.c_int32(k), None, C.c_int64(0))
            buf = C.create_string_buffer(int(n) + 1)
            self.lib.b200aln_batch_get_cigar(self.h, C.c_int32(k), buf, C.c_int64(int(n) + 1))
            out.append((buf.value, int(ed.value)))
        return out

    def ops(self, k: int) -> np.ndarray:
        """Alignment::get_alignment() of alignment k as edlib operation codes (0 match, 1 insert, 2 delete, 3 mismatch)."""
        n = self.lib.b200aln_batch_get_ops(self.h, C.c_int32(k), None, C.c_int64(0))
        if n < 0:
            raise RuntimeError(f"alignment {k}: {status_string(-n)}")
        out = np.zeros(int(n) + 1, dtype=np.uint8)
        self.lib.b200aln_batch_get_ops(self.h, C.c_int32(k), out.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_int64(int(n)))
        return out[:int(n)]

    def info(self) -> dict:
        bi = AlnBatchInfo()
        self.lib.b200aln_batch_get_info(self.h, C.byref(bi))
        return bi.as_dict()

    def reset(self):
        self.lib.b200aln_batch_reset(self.h)

    def split_log(self) -> np.ndarray:
        """Test build only (racon_gpu_b200/variants/libb200poa_digest.so): the split log of the last align_all, one
        SPLIT_REC_DTYPE record per split attempt.  Raises when the log overflowed."""
        return self._debug_log("b200aln_debug_split_log", SPLIT_REC_DTYPE, "split")

    def leaf_log(self) -> np.ndarray:
        """Test build only: the leaf log of the last align_all, one LEAF_REC_DTYPE record per leaf.  Raises when the log
        overflowed."""
        return self._debug_log("b200aln_debug_leaf_log", LEAF_REC_DTYPE, "leaf")

    def _debug_log(self, name, dtype, what) -> np.ndarray:
        fn = getattr(self.lib, name, None)
        if fn is None:
            raise RuntimeError(f"this library has no {what} log: load the digest build")
        count, rec_bytes = C.c_int64(0), C.c_int32(0)
        st = fn(self.h, None, C.c_int64(0), C.byref(count), C.byref(rec_bytes))
        if st not in (SUCCESS, GENERIC_ERROR):
            raise RuntimeError(f"{name}: {status_string(st)}")
        assert rec_bytes.value == dtype.itemsize, (rec_bytes.value, dtype.itemsize)
        out = np.zeros(count.value, dtype=dtype)
        st = fn(self.h, out.ctypes.data_as(C.c_void_p), C.c_int64(count.value), C.byref(count), C.byref(rec_bytes))
        if st == GENERIC_ERROR:
            raise RuntimeError(f"the {what} log overflowed: {count.value} records appended")
        if st != SUCCESS:
            raise RuntimeError(f"{name}: {status_string(st)}")
        return out


def pack_pairs(pairs):
    """[(query, target)] -> the columnar form b200aln_align_pairs takes."""
    q = np.frombuffer(b"".join(p[0] for p in pairs), dtype=np.uint8)
    t = np.frombuffer(b"".join(p[1] for p in pairs), dtype=np.uint8)
    q_off = np.zeros(len(pairs) + 1, dtype=np.int64)
    t_off = np.zeros(len(pairs) + 1, dtype=np.int64)
    np.cumsum([len(p[0]) for p in pairs], out=q_off[1:])
    np.cumsum([len(p[1]) for p in pairs], out=t_off[1:])
    return np.ascontiguousarray(q), q_off, np.ascontiguousarray(t), t_off


def align_pairs(q, q_off, t, t_off, device_id: int = 0, max_gpu_memory: int = 0, cigar_cap: int | None = None):
    """b200aln_align_pairs: (edit distances, cigar bytes, cigar offsets, info dict)."""
    lib = _lib()
    n = len(q_off) - 1
    if cigar_cap is None:
        cigar_cap = int(q_off[-1] + t_off[-1]) * 2 + 16 * n + 64
    ed = np.zeros(max(n, 1), dtype=np.int32)
    cigars = np.zeros(cigar_cap, dtype=np.uint8)
    coff = np.zeros(n + 1, dtype=np.int64)
    bi = AlnBatchInfo()
    p = lambda a, ty: a.ctypes.data_as(C.POINTER(ty))
    st = lib.b200aln_align_pairs(C.c_int32(device_id), C.c_int64(int(max_gpu_memory)), C.c_int64(n), p(q, C.c_uint8),
                                 p(q_off, C.c_int64), p(t, C.c_uint8), p(t_off, C.c_int64), p(ed, C.c_int32),
                                 p(cigars, C.c_char), C.c_int64(cigar_cap), p(coff, C.c_int64), C.byref(bi))
    if st != SUCCESS:
        raise RuntimeError(f"b200aln_align_pairs: {status_string(st)}")
    return ed[:n], cigars, coff, bi.as_dict()


class AlignerPool:
    """b200aln_aligner_*: batches_per_device batches on every listed device, one host thread per batch -- the GPU section
    of CUDAPolisher::find_overlap_breaking_points (src/cuda/cudapolisher.cpp:74-214) over columnar segments."""

    def __init__(self, devices=(0,), batches_per_device: int = 2, max_gpu_memory_per_batch: int = 0):
        self.lib = _lib()
        self.h = C.c_void_p()
        dev = (C.c_int32 * len(devices))(*devices)
        st = self.lib.b200aln_aligner_create(C.c_int32(len(devices)), dev, C.c_int32(batches_per_device),
                                             C.c_int64(int(max_gpu_memory_per_batch)), C.byref(self.h))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_aligner_create: {status_string(st)}")
        self._buf = np.zeros(0, dtype=np.uint8)

    def close(self):
        if self.h:
            self.lib.b200aln_aligner_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def align(self, q, q_off, t, t_off):
        """(edit distances, cigar buffer, cigar_off, cigar_len, info dict); pair k's CIGAR = buffer[off[k] : off[k] + len[k]]."""
        n = len(q_off) - 1
        need = 2 * int(q_off[-1] + t_off[-1]) + 2 * n + 64  # "1M1I1M...": two characters an operation at worst (+ 0 bytes)
        if self._buf.shape[0] < need:
            self._buf = np.zeros(need, dtype=np.uint8)
        ed = np.zeros(max(n, 1), dtype=np.int32)
        off = np.zeros(max(n, 1), dtype=np.int64)
        ln = np.zeros(max(n, 1), dtype=np.int32)
        used = C.c_int64(0)
        bi = AlnBatchInfo()
        p = lambda a, ty: a.ctypes.data_as(C.POINTER(ty))
        st = self.lib.b200aln_aligner_align(self.h, C.c_int64(n), p(q, C.c_uint8), p(q_off, C.c_int64), p(t, C.c_uint8),
                                            p(t_off, C.c_int64), p(ed, C.c_int32), p(self._buf, C.c_char),
                                            C.c_int64(self._buf.shape[0]), p(off, C.c_int64), p(ln, C.c_int32),
                                            C.byref(used), C.byref(bi))
        if st != SUCCESS:
            raise RuntimeError(f"b200aln_aligner_align: {status_string(st)}")
        return ed[:n], self._buf, off[:n], ln[:n], bi.as_dict()


class pinned:
    """Context manager: page-lock numpy arrays for the duration (b200aln_host_register / _unregister)."""

    def __init__(self, *arrays):
        self.arrays = [a for a in arrays if a.nbytes > 0]
        self.done = []

    def __enter__(self):
        lib = _lib()
        for a in self.arrays:
            st = lib.b200aln_host_register(C.c_void_p(a.ctypes.data), C.c_int64(a.nbytes))
            if st != SUCCESS:
                self.__exit__(None, None, None)
                raise RuntimeError(f"b200aln_host_register: {status_string(st)}")
            self.done.append(a)
        return self

    def __exit__(self, *exc):
        lib = _lib()
        for a in self.done:
            lib.b200aln_host_unregister(C.c_void_p(a.ctypes.data))
        self.done = []
        return False
