"""ctypes binding of the C ABI (include/b200poa.h) and the Python mirror of racon's batch adapter.

`PoaBatch` wraps one `b200poa_batch` (== one `cudapoa::Batch`, vendor/GenomeWorks/
cudapoa/include/claraparabricks/genomeworks/cudapoa/batch.hpp:88-160).  `CUDABatchProcessor` mirrors
racon's adapter of the same name (src/cuda/cudabatch.cpp:41-278): addWindow ->
generateConsensus -> trimmed consensus + per-window status, but with the CPU path's trimming rule
(src/window.cpp:118-139), which is the parity target.

There is no CPU fallback anywhere in this module: if libb200poa.so cannot be built or loaded, or no
CUDA device is visible, it raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .windows import WindowBatch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("B200POA_LIB", os.path.join(_HERE, "libb200poa.so"))  # B200POA_LIB: experiments only

SUCCESS = 0
EXCEEDED_MAXIMUM_POAS = 1
EXCEEDED_MAXIMUM_SEQUENCE_SIZE = 2
EXCEEDED_MAXIMUM_SEQUENCES_PER_POA = 3
PARTIAL_SPAN_UNSUPPORTED = 14
FULL_BAND = 0
STATIC_BAND = 1
ADAPTIVE_BAND = 2
OUTPUT_CONSENSUS = 1
OUTPUT_MSA = 2
OUTPUT_TYPE_UNAVAILABLE = 9

#: every symbol include/b200poa.h declares (tests check the library exports all of them)
ABI_SYMBOLS = (
    "b200poa_init", "b200poa_config_default", "b200poa_batch_create", "b200poa_batch_add_group",
    "b200poa_layer_order", "b200poa_batch_add_windows", "b200poa_batch_total_poas",
    "b200poa_batch_generate", "b200poa_batch_upload", "b200poa_batch_launch",
    "b200poa_batch_download", "b200poa_batch_get_consensus", "b200poa_batch_get_msa", "b200poa_batch_id",
    "b200poa_batch_reset", "b200poa_batch_destroy", "b200poa_batch_get_info", "b200poa_batch_set_option",
    "b200poa_polisher_create_ex", "b200poa_compact_rows", "b200poa_batch_add_windows_pinned", "b200poa_weight_modes",
    "b200poa_arena_append_columns",
    "b200poa_status_string", "b200poa_batch_phase_cycles", "b200poa_polish_windows", "b200poa_polish_windows_via_adapter",
    "b200poa_polisher_create", "b200poa_polisher_polish", "b200poa_polisher_destroy",
    "b200poa_arena_create", "b200poa_arena_add_window", "b200poa_arena_add_layer", "b200poa_arena_finalize",
    "b200poa_arena_view", "b200poa_polisher_polish_arena", "b200poa_arena_destroy",
    "b200poa_batch_add_windows_from_aligner", "b200poa_polish_overlaps", "b200poa_polish_overlaps_ex",
    "b200poa_free_export", "b200poa_polish_overlaps_multi",
)


class Config(C.Structure):
    _fields_ = [("max_sequence_size", C.c_int32), ("max_consensus_size", C.c_int32),
                ("max_nodes_per_graph", C.c_int32), ("alignment_band_width", C.c_int32),
                ("max_sequences_per_poa", C.c_int32), ("band_mode", C.c_int32)]


class Entry(C.Structure):
    _fields_ = [("seq", C.c_char_p), ("weights", C.POINTER(C.c_int8)), ("length", C.c_int32),
                ("begin", C.c_int32), ("end", C.c_int32)]


class BatchInfo(C.Structure):
    _fields_ = [("n_slots", C.c_int32), ("max_poas", C.c_int32), ("arena_capacity", C.c_int64),
                ("slot_bytes", C.c_int64), ("device_bytes", C.c_int64), ("staged_bases", C.c_int64),
                ("kernel_launches", C.c_int64), ("smem_bytes", C.c_int32), ("blocks_per_sm", C.c_int32),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64)]


class PolisherOptions(C.Structure):
    _fields_ = [("n_devices", C.c_int32), ("device_ids", C.POINTER(C.c_int32)), ("batches_per_device", C.c_int32),
                ("mem_per_batch", C.c_size_t), ("banded", C.c_int32), ("match", C.c_int32), ("mismatch", C.c_int32),
                ("gap", C.c_int32), ("max_sequence_size", C.c_int32), ("max_sequences_per_poa", C.c_int32),
                ("band_width", C.c_int32), ("accept_truncated", C.c_int32)]


_lib = None


def load_library(build_if_missing: bool = True) -> C.CDLL:
    """Load libb200poa.so (building it in-tree with nvcc if needed).  Raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from . import build as _build
        if _build.needs_build():
            _build.build()
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(f"{_LIB_PATH} is missing: build it with `python -m racon_gpu_b200.build` "
                           "(the POA engine has no CPU fallback)")
    lib = C.CDLL(_LIB_PATH)
    lib.b200poa_status_string.restype = C.c_char_p
    lib.b200poa_batch_destroy.restype = None
    lib.b200poa_config_default.restype = None
    lib.b200poa_layer_order.restype = None
    _lib = lib
    return lib


def _band_mode(banded) -> int:
    if banded == "adaptive" or banded == ADAPTIVE_BAND and banded is not True:
        return ADAPTIVE_BAND
    return STATIC_BAND if banded else FULL_BAND


def status_string(st: int) -> str:
    return load_library().b200poa_status_string(C.c_int32(int(st))).decode()


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


def layer_order(begins: np.ndarray) -> np.ndarray:
    """Processing order of a window's sequences (src/window.cpp:78-85)."""
    begins = np.ascontiguousarray(begins, dtype=np.int32)
    out = np.zeros(begins.shape[0], dtype=np.int32)
    load_library().b200poa_layer_order(C.c_int32(begins.shape[0]), _p(begins, C.c_int32), _p(out, C.c_int32))
    return out


def processing_order(batch: WindowBatch) -> np.ndarray:
    order = np.zeros(batch.n_seqs, dtype=np.int32)
    for w in range(batch.n_windows):
        s0, s1 = int(batch.win_seq_off[w]), int(batch.win_seq_off[w + 1])
        order[s0:s1] = layer_order(batch.begins[s0:s1])
    return order


class PoaBatch:
    """One `b200poa_batch`.  `stream` is a raw cudaStream_t (int) owned by the caller, 0 = default."""

    def __init__(self, device: int = 0, stream: int = 0, max_gpu_mem: int = 8 << 30,
                 max_sequence_size: int = 1023, max_sequences_per_poa: int = 200,
                 band_width: int = 256, banded=False, gap: int = -4, mismatch: int = -5,
                 match: int = 3, output_mask: int = OUTPUT_CONSENSUS):
        """banded: False = full band, True = static band, "adaptive" = adaptive band (retry with twice the width)."""
        self.lib = load_library()
        self.cfg = Config()
        self.lib.b200poa_config_default(C.byref(self.cfg), C.c_int32(max_sequence_size),
                                        C.c_int32(max_sequences_per_poa), C.c_int32(band_width),
                                        C.c_int32(_band_mode(banded)))
        self.handle = C.c_void_p()
        st = self.lib.b200poa_batch_create(C.c_int32(device), C.c_void_p(stream), C.c_size_t(max_gpu_mem),
                                           C.c_int32(output_mask), C.byref(self.cfg), C.c_int16(gap),
                                           C.c_int16(mismatch), C.c_int16(match), C.byref(self.handle))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_batch_create failed: {status_string(st)}")

    def close(self):
        if getattr(self, "handle", None) and self.handle.value:
            self.lib.b200poa_batch_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- cudapoa::Batch method set -------------------------------------------------------------
    def add_poa_group(self, entries):
        """entries: list of (seq: bytes, weights: np.int8 array | None[, begin, end]) in processing
        order.  Returns (status, per_seq_status list)."""
        n = len(entries)
        arr = (Entry * n)()
        keep = []
        for i, e in enumerate(entries):
            seq, wt = e[0], e[1]
            bg, en = (e[2], e[3]) if len(e) >= 4 else (-1, -1)
            arr[i].seq = seq
            if wt is None:
                arr[i].weights = C.cast(None, C.POINTER(C.c_int8))
            else:
                wt = np.ascontiguousarray(wt, dtype=np.int8)
                keep.append(wt)
                arr[i].weights = _p(wt, C.c_int8)
            arr[i].length = len(seq)
            arr[i].begin = bg
            arr[i].end = en
        per = np.zeros(n, dtype=np.int32)
        st = self.lib.b200poa_batch_add_group(self.handle, arr, C.c_int32(n), _p(per, C.c_int32))
        return st, per.tolist()

    def add_windows(self, batch: WindowBatch, first: int = 0):
        """Columnar add: stage windows [first, ...) until full.  Returns (n_added, seqs_added)."""
        n_added = C.c_int64(0)
        seqs_added = np.zeros(max(batch.n_windows - first, 1), dtype=np.int32)
        st = self.lib.b200poa_batch_add_windows(
            self.handle, C.c_int64(batch.n_windows), C.c_int64(first), _p(batch.win_seq_off, C.c_int64),
            _p(batch.seq_off, C.c_int64), _p(batch.bases, C.c_uint8), _p(batch.weights, C.c_int8),
            _p(batch.has_weights, C.c_uint8), _p(batch.begins, C.c_int32), _p(batch.ends, C.c_int32),
            C.byref(n_added), _p(seqs_added, C.c_int32))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_batch_add_windows failed: {status_string(st)}")
        return int(n_added.value), seqs_added[:n_added.value]

    def add_windows_from_aligner(self, aligner, bb_off: np.ndarray, bb_bases: np.ndarray, bb_qual=None, first: int = 0,
                                 last: int | None = None):
        """b200poa_batch_add_windows_from_aligner: windows [first, ...) of the aligner batch's window range, their
        layers gathered on the device from its arena; backbone w = bb_bases[bb_off[w]:bb_off[w + 1]] with qualities
        bb_qual (None: a FASTA target, weight 0).  The aligner must outlive this batch's results.  Returns
        (n_added, seqs_added)."""
        n_added = C.c_int64(0)
        bb_off = np.ascontiguousarray(bb_off, dtype=np.int64)
        seqs_added = np.zeros(max(bb_off.shape[0] - 1 - first, 1), dtype=np.int32)
        q = None if bb_qual is None else _p(np.ascontiguousarray(bb_qual, dtype=np.uint8), C.c_uint8)
        st = self.lib.b200poa_batch_add_windows_from_aligner(
            self.handle, aligner.h, C.c_int64(first), C.c_int64(bb_off.shape[0] - 1 if last is None else last),
            _p(bb_off, C.c_int64),
            _p(np.ascontiguousarray(bb_bases, dtype=np.uint8), C.c_uint8), q, C.byref(n_added), _p(seqs_added, C.c_int32))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_batch_add_windows_from_aligner failed: {status_string(st)}")
        return int(n_added.value), seqs_added[:n_added.value]

    def get_total_poas(self) -> int:
        return int(self.lib.b200poa_batch_total_poas(self.handle))

    def _check(self, st, what):
        if st != SUCCESS:
            raise RuntimeError(f"{what} failed: {status_string(st)}")

    def generate_poa(self):
        self._check(self.lib.b200poa_batch_generate(self.handle), "b200poa_batch_generate")

    def upload(self):
        self._check(self.lib.b200poa_batch_upload(self.handle), "b200poa_batch_upload")

    def launch(self):
        self._check(self.lib.b200poa_batch_launch(self.handle), "b200poa_batch_launch")

    def download(self):
        self._check(self.lib.b200poa_batch_download(self.handle), "b200poa_batch_download")

    def get_consensus(self, with_trim: bool = False):
        """Synchronises.  Returns (consensus list[bytes], coverage list[np.uint16], status np.int32) of the windows
        in add order (untrimmed); with_trim adds the device-side trim spans [(first, last)] (window.cpp:118-139)."""
        cons = C.POINTER(C.c_uint8)()
        cov = C.POINTER(C.c_uint16)()
        lens = C.POINTER(C.c_int32)()
        stat = C.POINTER(C.c_int32)()
        offs = C.POINTER(C.c_int32)()
        trim = C.POINTER(C.c_int32)()
        self._check(self.lib.b200poa_batch_get_consensus(self.handle, C.byref(cons), C.byref(cov), C.byref(lens),
                                                         C.byref(stat), C.byref(offs), C.byref(trim)),
                    "b200poa_batch_get_consensus")
        n = self.get_total_poas()
        if n == 0:
            return ([], [], np.zeros(0, dtype=np.int32)) + (([],) if with_trim else ())
        lens_a = np.ctypeslib.as_array(lens, shape=(n,)).copy()
        stat_a = np.ctypeslib.as_array(stat, shape=(n,)).copy()
        offs_a = np.ctypeslib.as_array(offs, shape=(n,)).copy()
        trim_a = np.ctypeslib.as_array(trim, shape=(n,)).copy()
        used = int((offs_a + lens_a).max())
        cons_a = np.ctypeslib.as_array(cons, shape=(max(used, 1),))
        out_c = [cons_a[offs_a[i]:offs_a[i] + lens_a[i]].tobytes() for i in range(n)]
        if cov:
            cov_a = np.ctypeslib.as_array(cov, shape=(max(used, 1),))
            out_v = [cov_a[offs_a[i]:offs_a[i] + lens_a[i]].copy() for i in range(n)]
        else:
            out_v = [None] * n
        if with_trim:
            return out_c, out_v, stat_a, [(int(t) & 0xFFFF, int(t) >> 16) for t in trim_a]
        return out_c, out_v, stat_a

    def get_msa(self):
        """Batch::get_msa.  Synchronises.  Returns (msa, status): msa[i] is the list of rows (bytes, one per staged
        sequence, in the order they were staged) of window i, or None where status[i] != 0."""
        msa = C.POINTER(C.c_uint8)()
        offs = C.POINTER(C.c_int64)()
        rows = C.POINTER(C.c_int32)()
        cols = C.POINTER(C.c_int32)()
        stat = C.POINTER(C.c_int32)()
        st = self.lib.b200poa_batch_get_msa(self.handle, C.byref(msa), C.byref(offs), C.byref(rows), C.byref(cols),
                                            C.byref(stat))
        if st == OUTPUT_TYPE_UNAVAILABLE:
            raise RuntimeError("b200poa_batch_get_msa: output_type_unavailable (create the batch with OUTPUT_MSA)")
        self._check(st, "b200poa_batch_get_msa")
        n = self.get_total_poas()
        if n == 0:
            return [], np.zeros(0, dtype=np.int32)
        offs_a = np.ctypeslib.as_array(offs, shape=(n,)).copy()
        rows_a = np.ctypeslib.as_array(rows, shape=(n,)).copy()
        cols_a = np.ctypeslib.as_array(cols, shape=(n,)).copy()
        stat_a = np.ctypeslib.as_array(stat, shape=(n,)).copy()
        used = int((offs_a + rows_a.astype(np.int64) * cols_a).max())
        arena = np.ctypeslib.as_array(msa, shape=(max(used, 1),)) if used > 0 else np.zeros(1, dtype=np.uint8)
        out = []
        for i in range(n):
            if stat_a[i] != SUCCESS:
                out.append(None)
                continue
            o, c = int(offs_a[i]), int(cols_a[i])
            out.append([arena[o + k * c:o + (k + 1) * c].tobytes() for k in range(int(rows_a[i]))])
        return out, stat_a

    def set_option(self, option: int, value: int):
        self._check(self.lib.b200poa_batch_set_option(self.handle, C.c_int32(option), C.c_int64(value)),
                    "b200poa_batch_set_option")

    def batch_id(self) -> int:
        return int(self.lib.b200poa_batch_id(self.handle))

    def reset(self):
        self.lib.b200poa_batch_reset(self.handle)

    def phase_cycles(self):
        """Diagnostics (B200POA_PHASE_TIMERS=1): dict phase -> summed cycles."""
        out = np.zeros(7, dtype=np.uint64)
        st = self.lib.b200poa_batch_phase_cycles(self.handle, _p(out, C.c_uint64), C.c_int32(7))
        if st != SUCCESS:
            return None
        names = ["program", "fill", "traceback", "add_alignment", "topsort", "consensus", "other"]
        return dict(zip(names, out.tolist()))

    def info(self) -> dict:
        inf = BatchInfo()
        self.lib.b200poa_batch_get_info(self.handle, C.byref(inf))
        return {k: getattr(inf, k) for k, _ in BatchInfo._fields_}


def trim_consensus(cons: bytes, cov: np.ndarray, n_seqs: int):
    """racon's TGS coverage trim, CPU semantics (src/window.cpp:118-139).
    Returns (consensus, chimeric_warning)."""
    avg = (n_seqs - 1) // 2
    ok = np.nonzero(cov >= avg)[0]
    if ok.shape[0] == 0:
        return cons, True
    b, e = int(ok[0]), int(ok[-1])
    if b >= e:
        return cons, True
    return cons[b:e + 1], False


class CUDABatchProcessor:
    """Python mirror of racon::CUDABatchProcessor (src/cuda/cudabatch.cpp) over a columnar arena.

    Differences from the reference adapter, all on purpose (SURVEY.md 8a-a7): the trim threshold,
    the chimeric-window status and the NGS status follow the CPU path (src/window.cpp:65-142), so a
    window this class reports `True` for is byte-identical to racon's CPU consensus.
    """

    def __init__(self, max_window_depth: int = 200, device: int = 0, avail_mem: int = 8 << 30,
                 gap: int = -4, mismatch: int = -5, match: int = 3, cuda_banded_alignment: bool = False,
                 stream: int = 0, tgs: bool = True, trim: bool = True):
        # cudabatch.cpp:56-68: BatchConfig(1023, max_window_depth, 256, band mode)
        self.batch = PoaBatch(device=device, stream=stream, max_gpu_mem=avail_mem,
                              max_sequence_size=1023, max_sequences_per_poa=max_window_depth,
                              band_width=256, banded=cuda_banded_alignment, gap=gap,
                              mismatch=mismatch, match=match)
        self.tgs, self.trim = tgs, trim
        self.n_seqs, self.seqs_added, self.backbones = [], [], []

    def add_windows(self, windows: WindowBatch, first: int = 0) -> int:
        """The addWindow loop of cudapolisher.cpp:254-276.  Returns how many windows fitted."""
        n, seqs_added = self.batch.add_windows(windows, first)
        s = windows.win_seq_off
        self.n_seqs.extend((s[first + 1:first + n + 1] - s[first:first + n]).tolist())
        self.seqs_added.extend(np.asarray(seqs_added).tolist())
        for w in range(first, first + n):  # the backbone, for windows that come back unpolished
            a, b = int(windows.seq_off[s[w]]), int(windows.seq_off[s[w] + 1])
            self.backbones.append(windows.bases[a:b].tobytes())
        return n

    def has_windows(self) -> bool:
        return self.batch.get_total_poas() > 0

    def generate_consensus(self):
        """Returns (list of consensus bytes, list of bool status) for the windows in the batch.  A window reported
        False holds its backbone: fewer than 3 sequences (window.cpp:68-71), a kernel status, or layers dropped by the
        batch limits (same rule as cuda_polisher.cpp / cuda_batch.cpp: left to the caller's CPU path)."""
        self.batch.generate_poa()
        cons, cov, status = self.batch.get_consensus()
        out, ok = [], []
        for i in range(len(cons)):
            if self.n_seqs[i] < 3 or status[i] != SUCCESS or self.seqs_added[i] != self.n_seqs[i] - 1:
                out.append(self.backbones[i])
                ok.append(False)
                continue
            c = cons[i]
            if self.tgs and self.trim:
                c, _ = trim_consensus(c, cov[i], self.n_seqs[i])
            out.append(c)
            ok.append(True)
        return out, ok

    def reset(self):
        self.batch.reset()
        self.n_seqs, self.seqs_added, self.backbones = [], [], []


def polish_windows(windows: WindowBatch, match: int = 3, mismatch: int = -5, gap: int = -4,
                   banded: bool = False, tgs: bool = True, trim: bool = True, devices=None,
                   batches_per_device: int = 1, mem_per_batch: int = 0, max_windows_per_round: int = 0,
                   stride: int = 2048, via_adapter: bool = False):
    """Whole-job call with HOST buffers (b200poa_polish_windows): racon's GPU window scheduler
    (src/cuda/cudapolisher.cpp:216-345) over a columnar arena.

    Returns (cons uint8 [W, stride], cons_len int32 [W], polished bool [W], status int32 [W],
    kernel_launches)."""
    lib = load_library()
    W = windows.n_windows
    cons = np.zeros((W, stride), dtype=np.uint8)
    clen = np.zeros(W, dtype=np.int32)
    pol = np.zeros(W, dtype=np.uint8)
    status = np.zeros(W, dtype=np.int32)
    dev = np.asarray(devices if devices is not None else [], dtype=np.int32)
    launches = C.c_int64(0)
    if via_adapter:  # the C++ class API mirroring racon's Window / CUDABatchProcessor / polish()
        st = lib.b200poa_polish_windows_via_adapter(
            C.c_int64(W), _p(windows.win_seq_off, C.c_int64), _p(windows.seq_off, C.c_int64),
            _p(windows.bases, C.c_uint8), _p(windows.weights, C.c_int8), _p(windows.has_weights, C.c_uint8),
            _p(windows.begins, C.c_int32), _p(windows.ends, C.c_int32), C.c_int32(int(tgs)), C.c_int32(int(trim)),
            C.c_int32(match), C.c_int32(mismatch), C.c_int32(gap), C.c_int32(int(banded)),
            C.c_int32(dev.shape[0]), _p(dev, C.c_int32) if dev.shape[0] else None, C.c_int32(batches_per_device),
            C.c_size_t(mem_per_batch), C.c_int32(max_windows_per_round), _p(cons, C.c_uint8), C.c_int32(stride),
            _p(clen, C.c_int32), _p(pol, C.c_uint8))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_polish_windows_via_adapter failed: {status_string(st)}")
        return cons, clen, pol.astype(bool), status, 0
    st = lib.b200poa_polish_windows(
        C.c_int64(W), _p(windows.win_seq_off, C.c_int64), _p(windows.seq_off, C.c_int64),
        _p(windows.bases, C.c_uint8), _p(windows.weights, C.c_int8), _p(windows.has_weights, C.c_uint8),
        _p(windows.begins, C.c_int32), _p(windows.ends, C.c_int32), C.c_int32(int(tgs)), C.c_int32(int(trim)),
        C.c_int32(match), C.c_int32(mismatch), C.c_int32(gap), C.c_int32(int(banded)),
        C.c_int32(dev.shape[0]), _p(dev, C.c_int32) if dev.shape[0] else None, C.c_int32(batches_per_device),
        C.c_size_t(mem_per_batch), C.c_int32(max_windows_per_round), _p(cons, C.c_uint8), C.c_int32(stride),
        _p(clen, C.c_int32), _p(pol, C.c_uint8), _p(status, C.c_int32), C.byref(launches))
    if st != SUCCESS:
        raise RuntimeError(f"b200poa_polish_windows failed: {status_string(st)}")
    return cons, clen, pol.astype(bool), status, int(launches.value)


def compact_rows(cons: np.ndarray, clen: np.ndarray, flat: np.ndarray | None = None):
    """Rows of a [W, stride] consensus matrix packed back to back (b200poa_compact_rows).  Returns (flat, offsets)."""
    lib = load_library()
    lib.b200poa_compact_rows.restype = C.c_int64
    W, stride = cons.shape
    clen = np.ascontiguousarray(clen, dtype=np.int32)
    total = int(np.minimum(clen, stride).sum())
    if flat is None or flat.shape[0] < total:
        flat = np.empty(max(total, 1), dtype=np.uint8)
    off = np.zeros(W + 1, dtype=np.int64)
    n = lib.b200poa_compact_rows(_p(cons, C.c_uint8), C.c_int64(W), C.c_int64(stride), _p(clen, C.c_int32),
                                 _p(flat, C.c_uint8), _p(off, C.c_int64))
    return flat[:n], off


def consensus_list(cons: np.ndarray, clen: np.ndarray):
    return [cons[w, :clen[w]].tobytes() for w in range(cons.shape[0])]


class Polisher:
    """Persistent GPU window polisher (b200poa_polisher_*): batch processors are created once and
    reused by every `polish` call, like one `CUDAPolisher::polish` run does (cudapolisher.cpp:226-240)."""

    def __init__(self, devices=None, batches_per_device: int = 1, mem_per_batch: int = 0, banded: bool = False,
                 match: int = 3, mismatch: int = -5, gap: int = -4, max_sequence_size: int = 0,
                 max_sequences_per_poa: int = 0, band_width: int = 0, accept_truncated: bool = False):
        self.lib = load_library()
        self.lib.b200poa_polisher_destroy.restype = None
        dev = np.asarray(devices if devices is not None else [], dtype=np.int32)
        self.handle = C.c_void_p()
        opt = PolisherOptions(dev.shape[0], _p(dev, C.c_int32) if dev.shape[0] else None, batches_per_device,
                              mem_per_batch, _band_mode(banded), match, mismatch, gap, max_sequence_size,
                              max_sequences_per_poa, band_width, int(accept_truncated))
        st = self.lib.b200poa_polisher_create_ex(C.byref(opt), C.byref(self.handle))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_polisher_create_ex failed: {status_string(st)}")
        self.last = {}

    def polish(self, windows: WindowBatch, tgs: bool = True, trim: bool = True, max_windows_per_round: int = 0,
               stride: int = 2048, out=None):
        """Returns (cons [W, stride] uint8, cons_len, polished, status).  `out` lets the caller reuse
        output arrays between calls."""
        W = windows.n_windows
        if out is None:
            out = (np.zeros((W, stride), dtype=np.uint8), np.zeros(W, dtype=np.int32),
                   np.zeros(W, dtype=np.uint8), np.zeros(W, dtype=np.int32))
        cons, clen, pol, status = out
        launches, h2d, d2h = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        st = self.lib.b200poa_polisher_polish(
            self.handle, C.c_int64(W), _p(windows.win_seq_off, C.c_int64), _p(windows.seq_off, C.c_int64),
            _p(windows.bases, C.c_uint8), _p(windows.weights, C.c_int8), _p(windows.has_weights, C.c_uint8),
            _p(windows.begins, C.c_int32), _p(windows.ends, C.c_int32), C.c_int32(int(tgs)), C.c_int32(int(trim)),
            C.c_int32(max_windows_per_round), _p(cons, C.c_uint8), C.c_int32(stride), _p(clen, C.c_int32),
            _p(pol, C.c_uint8), _p(status, C.c_int32), C.byref(launches), C.byref(h2d), C.byref(d2h))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_polisher_polish failed: {status_string(st)}")
        self.last = {"kernel_launches": int(launches.value), "h2d_bytes": int(h2d.value), "d2h_bytes": int(d2h.value)}
        return cons, clen, pol.astype(bool), status

    def polish_arena(self, arena: "WindowArena", tgs: bool = True, trim: bool = True, max_windows_per_round: int = 0,
                     stride: int = 2048, out=None):
        """`polish` over windows built with WindowArena (b200poa_polisher_polish_arena).  The finalized arena is
        page-locked: every batch uploads its byte range straight from it, no staging copy on the host."""
        W = arena.n_windows
        if out is None:
            out = (np.zeros((W, stride), dtype=np.uint8), np.zeros(W, dtype=np.int32),
                   np.zeros(W, dtype=np.uint8), np.zeros(W, dtype=np.int32))
        cons, clen, pol, status = out
        launches, h2d, d2h = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        st = self.lib.b200poa_polisher_polish_arena(
            self.handle, arena.handle, C.c_int32(int(tgs)), C.c_int32(int(trim)), C.c_int32(max_windows_per_round),
            _p(cons, C.c_uint8), C.c_int32(stride), _p(clen, C.c_int32), _p(pol, C.c_uint8), _p(status, C.c_int32),
            C.byref(launches), C.byref(h2d), C.byref(d2h))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_polisher_polish_arena failed: {status_string(st)}")
        self.last = {"kernel_launches": int(launches.value), "h2d_bytes": int(h2d.value), "d2h_bytes": int(d2h.value)}
        return cons, clen, pol.astype(bool), status

    def close(self):
        if getattr(self, "handle", None) and self.handle.value:
            self.lib.b200poa_polisher_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class WindowArena:
    """Columnar window construction (b200poa_arena_*): racon's createWindow / Window::add_layer contract
    (src/window.cpp:15-63) writing into the arena the engine consumes.  Host-only, needs no GPU.
    Sequences are `bytes`; the object keeps them alive until `finalize` (the C side borrows the pointers)."""

    def __init__(self):
        self.lib = load_library()
        self.lib.b200poa_arena_create.restype = C.c_void_p
        self.lib.b200poa_arena_add_window.restype = C.c_int64
        self.lib.b200poa_arena_destroy.restype = None
        self.handle = C.c_void_p(self.lib.b200poa_arena_create())
        self._keep = []
        self.n_windows = 0

    def add_window(self, backbone: bytes, quality: bytes) -> int:
        self._keep += [backbone, quality]
        w = int(self.lib.b200poa_arena_add_window(self.handle, C.c_char_p(backbone), C.c_uint32(len(backbone)),
                                                  C.c_char_p(quality), C.c_uint32(len(quality) if quality is not None else 0)))
        if w >= 0:
            self.n_windows = w + 1
        return w

    def add_layer(self, window: int, sequence: bytes, quality, begin: int, end: int) -> bool:
        self._keep += [sequence, quality]
        st = self.lib.b200poa_arena_add_layer(self.handle, C.c_int64(window), C.c_char_p(sequence), C.c_uint32(len(sequence)),
                                              C.c_char_p(quality) if quality is not None else None,
                                              C.c_uint32(len(quality) if quality is not None else 0),
                                              C.c_uint32(begin), C.c_uint32(end))
        return st == SUCCESS

    @classmethod
    def from_batch(cls, batch: WindowBatch) -> "WindowArena":
        """An arena holding the windows of a columnar batch (b200poa_arena_append_columns), finalized."""
        a = cls()
        st = a.lib.b200poa_arena_append_columns(
            a.handle, C.c_int64(batch.n_windows), _p(batch.win_seq_off, C.c_int64), _p(batch.seq_off, C.c_int64),
            _p(batch.bases, C.c_uint8), _p(batch.weights, C.c_int8), _p(batch.has_weights, C.c_uint8),
            _p(batch.begins, C.c_int32), _p(batch.ends, C.c_int32))
        if st != SUCCESS:
            raise RuntimeError(f"b200poa_arena_append_columns failed: {status_string(st)}")
        a.n_windows = batch.n_windows
        a.finalize(view=False)
        return a

    def finalize(self, view: bool = True):
        """Group and copy (and page-lock, where a CUDA device exists); returns the arena as a WindowBatch (copies of the
        C arrays) unless view=False."""
        if self.lib.b200poa_arena_finalize(self.handle) != SUCCESS:
            raise RuntimeError("b200poa_arena_finalize failed")
        self._keep = []
        if not view:
            return None
        nw, ns = C.c_int64(0), C.c_int64(0)
        pw, ps = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
        pb, pwt, ph = C.POINTER(C.c_uint8)(), C.POINTER(C.c_int8)(), C.POINTER(C.c_uint8)()
        pbg, pen = C.POINTER(C.c_int32)(), C.POINTER(C.c_int32)()
        st = self.lib.b200poa_arena_view(self.handle, C.byref(nw), C.byref(ns), C.byref(pw), C.byref(ps), C.byref(pb),
                                         C.byref(pwt), C.byref(ph), C.byref(pbg), C.byref(pen))
        if st != SUCCESS:
            raise RuntimeError("b200poa_arena_view failed")
        W, S = int(nw.value), int(ns.value)

        def arr(ptr, n, dt):
            return np.ctypeslib.as_array(ptr, shape=(n,)).astype(dt, copy=True) if n else np.zeros(0, dtype=dt)
        seq_off = arr(ps, S + 1, np.int64)
        B = int(seq_off[-1]) if S else 0
        return WindowBatch(win_seq_off=arr(pw, W + 1, np.int64), seq_off=seq_off, bases=arr(pb, B, np.uint8),
                           weights=arr(pwt, B, np.int8), has_weights=arr(ph, S, np.uint8),
                           begins=arr(pbg, S, np.int32), ends=arr(pen, S, np.int32))

    def close(self):
        if getattr(self, "handle", None) and self.handle.value:
            self.lib.b200poa_arena_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class OverlapOptions(C.Structure):
    """include/b200poa.h b200poa_overlap_options"""
    _fields_ = [("device_id", C.c_int32), ("poa_batches", C.c_int32), ("mem_per_poa_batch", C.c_size_t),
                ("aligner_mem", C.c_int64), ("window_length", C.c_int32), ("quality_threshold", C.c_double),
                ("banded", C.c_int32), ("match", C.c_int32), ("mismatch", C.c_int32), ("gap", C.c_int32),
                ("tgs", C.c_int32), ("trim", C.c_int32), ("max_windows_per_batch", C.c_int32)]


class OverlapExport(C.Structure):
    """include/b200poa.h b200poa_overlap_export"""
    _fields_ = [("n_windows", C.c_int64), ("n_sequences", C.c_int64), ("window_ids", C.POINTER(C.c_int64)),
                ("win_seq_off", C.POINTER(C.c_int64)), ("seq_off", C.POINTER(C.c_int64)),
                ("bases", C.POINTER(C.c_uint8)), ("weights", C.POINTER(C.c_int8)),
                ("has_weights", C.POINTER(C.c_uint8)), ("begins", C.POINTER(C.c_int32)), ("ends", C.POINTER(C.c_int32))]


class OverlapEx(C.Structure):
    """include/b200poa.h b200poa_overlap_ex"""
    _fields_ = [("deep_windows", C.c_int32), ("export_layers", C.c_int32), ("deep_max_sequence_size", C.c_int32),
                ("deep_max_sequences_per_poa", C.c_int32), ("exported", OverlapExport),
                ("tier2_windows", C.c_int64), ("tier2_polished", C.c_int64), ("tier2_batches", C.c_int64),
                ("exported_windows", C.c_int64), ("exported_bytes", C.c_int64)]


def _export_batch(e: OverlapExport):
    """(window ids, WindowBatch) copied out of a b200poa_overlap_export"""
    W, S = int(e.n_windows), int(e.n_sequences)

    def arr(ptr, n, dt):
        return np.ctypeslib.as_array(ptr, shape=(n,)).astype(dt, copy=True) if n else np.zeros(0, dtype=dt)
    seq_off = arr(e.seq_off, S + 1, np.int64)
    B = int(seq_off[-1])
    return arr(e.window_ids, W, np.int64), WindowBatch(
        win_seq_off=arr(e.win_seq_off, W + 1, np.int64), seq_off=seq_off, bases=arr(e.bases, B, np.uint8),
        weights=arr(e.weights, B, np.int8), has_weights=arr(e.has_weights, S, np.uint8),
        begins=arr(e.begins, S, np.int32), ends=arr(e.ends, S, np.int32))


def polish_overlaps(t_bases, t_off, t_qual, t_id, t_begin, t_end, q_bases, q_off, q_qual, has_quality, q_first,
                    window_length=500, quality_threshold=10.0, match=3, mismatch=-5, gap=-4, banded=False, tgs=True,
                    trim=True, device=0, poa_batches=1, mem_per_poa_batch=0, aligner_mem=0, max_windows_per_batch=0,
                    stride=4096, deep_windows=False, export_layers=False, deep_max_sequence_size=0,
                    deep_max_sequences_per_poa=0, devices=None):
    """b200poa_polish_overlaps (racon_b200::polish_overlaps): contigs and racon's filtered overlaps in, per window
    (contig by contig) the consensus list, polished, status out, plus {"rounds", "h2d_bytes", "d2h_bytes"}.
    Raises when a contig's overlaps do not fit one aligner batch (the error names the contig).

    deep_windows: a second tier of POA batches polishes the windows racon's limits (200 sequences, 1023 bases) leave
    unpolished (b200poa_polish_overlaps_ex; deep_max_* cap that tier, 0 = the engine's limits).  export_layers: the
    windows still unpolished with at least 3 sequences come back as info["export"] = (window ids, WindowBatch in the
    layout of racon_gpu_b200/windows.py), ready for Polisher.polish or racon's CPU pass.  With either set, info also
    has "tier2_windows", "tier2_polished", "tier2_batches", "exported_windows" and "exported_bytes".

    devices: None runs on `device` alone, as above.  A list runs one worker per entry (b200poa_polish_overlaps_multi;
    [] = every visible device, an id listed twice = two workers on it) and splits a contig too large for one aligner
    batch at window boundaries; the outputs equal the single-device call's.  info["rounds"] then counts units, and info
    also has "split_contigs" (contigs polished in more than one unit) and "repeat_overlaps" (alignments done more than
    once because of the splits)."""
    lib = load_library()
    o = OverlapOptions(device, poa_batches, mem_per_poa_batch, aligner_mem, window_length, float(quality_threshold),
                       int(bool(banded)), match, mismatch, gap, int(tgs), int(trim), max_windows_per_batch)
    ex = None
    if deep_windows or export_layers or deep_max_sequence_size or deep_max_sequences_per_poa:
        ex = OverlapEx(int(bool(deep_windows)), int(bool(export_layers)), deep_max_sequence_size,
                       deep_max_sequences_per_poa)
    t_off = np.ascontiguousarray(t_off, dtype=np.int64)
    lens = np.diff(t_off)
    n_win = int(((lens + window_length - 1) // window_length).sum())
    cons = np.zeros((max(n_win, 1), stride), dtype=np.uint8)
    clen = np.zeros(max(n_win, 1), dtype=np.int32)
    pol = np.zeros(max(n_win, 1), dtype=np.uint8)
    st = np.zeros(max(n_win, 1), dtype=np.int32)
    rounds, h2d, d2h, unfit = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(-1)
    split, repeat = C.c_int64(0), C.c_int64(0)
    u8 = lambda a: None if a is None else _p(np.ascontiguousarray(a, dtype=np.uint8), C.c_uint8)
    keep = [np.ascontiguousarray(a, dtype=d) for a, d in ((t_bases, np.uint8), (q_bases, np.uint8),
                                                           (t_id, np.int32), (t_begin, np.int32), (t_end, np.int32),
                                                           (q_off, np.int64), (q_first, np.int32))]
    tq = None if t_qual is None else np.ascontiguousarray(t_qual, dtype=np.uint8)
    qq = None if q_qual is None else np.ascontiguousarray(q_qual, dtype=np.uint8)
    hq = None if has_quality is None else np.ascontiguousarray(has_quality, dtype=np.uint8)
    args = (C.c_int64(len(t_off) - 1), _p(keep[0], C.c_uint8), _p(t_off, C.c_int64), u8(tq),
            C.c_int64(len(keep[2])), _p(keep[2], C.c_int32), _p(keep[3], C.c_int32), _p(keep[4], C.c_int32),
            _p(keep[1], C.c_uint8), _p(keep[5], C.c_int64), u8(qq), u8(hq), _p(keep[6], C.c_int32),
            _p(cons, C.c_uint8), C.c_int32(stride), _p(clen, C.c_int32), _p(pol, C.c_uint8), _p(st, C.c_int32),
            C.byref(rounds), C.byref(h2d), C.byref(d2h), C.byref(unfit))
    if devices is not None:
        dev = np.ascontiguousarray(list(devices), dtype=np.int32)
        lib.b200poa_free_export.restype = None
        rc = lib.b200poa_polish_overlaps_multi(C.byref(o), None if ex is None else C.byref(ex), C.c_int32(len(dev)),
                                               _p(dev, C.c_int32) if len(dev) else None, *args, C.byref(split),
                                               C.byref(repeat))
        if ex is not None:
            exported = _export_batch(ex.exported) if rc == SUCCESS and export_layers else None
            lib.b200poa_free_export(C.byref(ex.exported))
    elif ex is None:
        rc = lib.b200poa_polish_overlaps(C.byref(o), *args)
    else:
        lib.b200poa_free_export.restype = None
        rc = lib.b200poa_polish_overlaps_ex(C.byref(o), C.byref(ex), *args)
        exported = _export_batch(ex.exported) if rc == SUCCESS and export_layers else None
        lib.b200poa_free_export(C.byref(ex.exported))
    if rc != SUCCESS:
        what = f" (contig {unfit.value} does not fit one aligner batch)" if unfit.value >= 0 else ""
        if devices is not None and unfit.value >= 0:
            what = f" (the overlaps of one window of contig {unfit.value} do not fit one aligner batch)"
        raise RuntimeError(f"b200poa_polish_overlaps failed: {status_string(rc)}{what}")
    out = [cons[i, :min(int(clen[i]), stride)].tobytes() for i in range(n_win)]
    info = {"rounds": int(rounds.value), "h2d_bytes": int(h2d.value), "d2h_bytes": int(d2h.value)}
    if devices is not None:
        info.update({"split_contigs": int(split.value), "repeat_overlaps": int(repeat.value)})
    if ex is not None:
        info.update({k: int(getattr(ex, k)) for k in ("tier2_windows", "tier2_polished", "tier2_batches",
                                                       "exported_windows", "exported_bytes")})
        if export_layers:
            info["export"] = exported
    return out, pol[:n_win].astype(bool), st[:n_win], info
