"""aho_corasick_b200 -- host-side mirror of the reference's search API over libacb200.so.

The names, argument meaning and error behaviour follow BurntSushi/aho-corasick 1.1.3
(`AhoCorasick`, `AhoCorasickBuilder`, `MatchKind`, `StartKind`, `AhoCorasickKind`, `Match`,
`find_iter`, `find_overlapping_iter`, `try_*`; src/ahocorasick.rs, src/lib.rs:239-251), so the
parity tests read like the reference's own.  Everything that touches a haystack goes through the
C ABI (include/acb200.h) into hand-written sm_90a kernels; there is no CPU search path here.
Python is test/bench glue only: the product is the shared library.
"""
from __future__ import annotations

import collections
import ctypes as C
import enum
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libacb200.so"


class NativeLibraryMissing(ImportError):
    pass


def _load():
    if not _LIB_PATH.exists():
        raise NativeLibraryMissing(
            f"{_LIB_PATH} is missing: build it with `python aho-corasick_b200/build.py` "
            "(nvcc, sm_90a). There is no fallback implementation.")
    return C.CDLL(str(_LIB_PATH))


_lib = _load()


class MatchKind(enum.IntEnum):  # src/util/search.rs:1052
    Standard = 0
    LeftmostFirst = 1
    LeftmostLongest = 2


class StartKind(enum.IntEnum):  # src/util/search.rs:1133
    Unanchored = 0
    Anchored = 1
    Both = 2


class AhoCorasickKind(enum.IntEnum):  # src/ahocorasick.rs:2624
    NoncontiguousNFA = 1
    ContiguousNFA = 2
    DFA = 3


class Anchored(enum.IntEnum):  # src/util/search.rs:784
    No = 0
    Yes = 1


class Engine(enum.IntEnum):
    Auto = 0
    Walk = 1
    Prefilter = 2
    Sequential = 3


E_OVERFLOW = -21


class BuildError(Exception):  # src/util/error.rs:23-49
    def __init__(self, code):
        super().__init__(_lib.acg_strerror(code).decode())
        self.code = code


class MatchError(Exception):  # src/util/error.rs:140-223
    def __init__(self, code):
        super().__init__(_lib.acg_strerror(code).decode())
        self.code = code

    @property
    def kind(self):
        return {-10: "InvalidInputAnchored", -11: "InvalidInputUnanchored", -12: "UnsupportedStream",
                -13: "UnsupportedOverlapping", -14: "UnsupportedEmpty"}.get(self.code, "Boundary")


class DeviceError(RuntimeError):
    def __init__(self, code):
        super().__init__(_lib.acg_strerror(code).decode())
        self.code = code


class _BuildOpts(C.Structure):
    _fields_ = [("match_kind", C.c_int32), ("start_kind", C.c_int32),
                ("ascii_case_insensitive", C.c_int32), ("byte_classes", C.c_int32),
                ("prefilter", C.c_int32), ("kind", C.c_int32), ("dense_depth", C.c_int64)]


class _Desc(C.Structure):
    _fields_ = [("trans", C.POINTER(C.c_uint32)), ("trans_len", C.c_uint64),
                ("stride2", C.c_uint32), ("alphabet_len", C.c_uint32),
                ("byte_classes", C.c_uint8 * 256),
                ("max_special_id", C.c_uint32), ("max_match_id", C.c_uint32),
                ("start_unanchored_id", C.c_uint32), ("start_anchored_id", C.c_uint32),
                ("match_offsets", C.POINTER(C.c_uint32)), ("match_pids", C.POINTER(C.c_uint32)),
                ("pattern_lens", C.POINTER(C.c_uint32)), ("n_patterns", C.c_uint32),
                ("match_kind", C.c_uint32), ("start_kind", C.c_uint32), ("prefilter_kind", C.c_uint32),
                ("min_pattern_len", C.c_uint64), ("max_pattern_len", C.c_uint64)]


class _Stats(C.Structure):
    _fields_ = [("engine", C.c_int32), ("launches", C.c_int32), ("candidates", C.c_uint64),
                ("raw_matches", C.c_uint64), ("scan_ms", C.c_float), ("order_ms", C.c_float),
                ("h2d_ms", C.c_float), ("d2h_ms", C.c_float)]


MATCH_DTYPE = np.dtype([("pid", "<u4"), ("_pad", "<u4"), ("start", "<u8"), ("end", "<u8")])
DOC_MATCH_DTYPE = np.dtype([("pid", "<u4"), ("doc", "<u4"), ("start", "<u8"), ("end", "<u8")])  # acg_doc_match

_vp, _u64, _i = C.c_void_p, C.c_uint64, C.c_int


def _declare(lib):
    """ctypes signatures of the C ABI (include/acb200.h)."""
    lib.acg_strerror.restype = C.c_char_p
    lib.acg_strerror.argtypes = [_i]
    lib.acg_build.argtypes = [C.POINTER(C.c_char_p), C.POINTER(_u64), _u64, C.POINTER(_BuildOpts), C.POINTER(_vp)]
    lib.acg_build_host.argtypes = lib.acg_build.argtypes
    lib.acg_build_on_device.argtypes = lib.acg_build.argtypes
    lib.acg_dfa_create.argtypes = [C.POINTER(_Desc), C.POINTER(_vp)]
    lib.acg_dfa_free.argtypes = [_vp]
    lib.acg_dfa_free.restype = None
    lib.acg_dfa_table.argtypes = [_vp, C.POINTER(_Desc)]
    for _f in ("acg_dfa_state_len", "acg_patterns_len", "acg_min_pattern_len", "acg_max_pattern_len",
               "acg_memory_usage"):
        getattr(lib, _f).argtypes = [_vp]
        getattr(lib, _f).restype = _u64
    for _f in ("acg_kind", "acg_match_kind", "acg_start_kind", "acg_prefilter_kind", "acg_last_engine"):
        getattr(lib, _f).argtypes = [_vp]
    lib.acg_packed_variant.argtypes = [_vp, C.POINTER(_i), C.POINTER(_i)]
    lib.acg_set_engine.argtypes = [_vp, _i]
    lib.acg_last_stats.argtypes = [_vp, C.POINTER(_Stats)]
    lib.acg_find_overlapping.argtypes = [_vp, _vp, _u64, _u64, _u64, _i, _vp, _u64, C.POINTER(_u64)]
    lib.acg_find_iter.argtypes = lib.acg_find_overlapping.argtypes
    lib.acg_find.argtypes = [_vp, _vp, _u64, _u64, _u64, _i, _i, _vp, C.POINTER(_i)]
    lib.acg_find_overlapping_dev.argtypes = [_vp, _vp, _u64, _u64, _u64, _vp, _u64, C.POINTER(_u64),
                                              C.POINTER(C.c_float)]
    lib.acg_find_iter_dev.argtypes = lib.acg_find_overlapping_dev.argtypes
    lib.acg_count_overlapping_dev.argtypes = [_vp, _vp, _u64, _u64, _u64, C.POINTER(_u64), C.POINTER(_u64),
                                               C.POINTER(C.c_float)]
    lib.acg_find_overlapping_devout.argtypes = [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _u64,
                                                 C.POINTER(_u64), C.POINTER(C.c_float)]
    lib.acg_find_iter_batch.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _i, _vp, _u64, C.POINTER(_u64)]
    lib.acg_find_overlapping_batch.argtypes = lib.acg_find_iter_batch.argtypes
    lib.acg_is_match_batch.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _i, _vp]
    lib.acg_find_batch.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _i, _i, _vp, _vp]
    lib.acg_find_iter_batch_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _i, _vp, _u64, _vp, C.POINTER(_u64)]
    lib.acg_find_overlapping_batch_devout.argtypes = lib.acg_find_iter_batch_devout.argtypes
    lib.acg_is_match_batch_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _i, _vp]
    lib.acg_find_batch_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _i, _i, _vp, _vp]
    lib.acg_pattern_counts_batch.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _i, _i, _vp, _vp, _vp, _u64,
                                             C.POINTER(_u64)]
    lib.acg_pattern_counts_batch_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _i, _i, _vp, _vp, _vp, _u64,
                                                    C.POINTER(_u64)]
    lib.acg_match_coverage_batch.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _i, _i, _vp, _vp]
    lib.acg_match_coverage_batch_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _i, _i, _vp, _vp]
    lib.acg_replace_all_batch.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _vp,
                                          C.POINTER(_u64)]
    lib.acg_replace_all_batch_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _vp, _vp, _u64, _vp, _u64, _vp,
                                                 C.POINTER(_u64)]
    lib.acg_streams_create.argtypes = [_vp, _u64, _i, C.POINTER(_vp)]
    lib.acg_streams_free.argtypes = [_vp]
    lib.acg_streams_free.restype = None
    lib.acg_streams_reset.argtypes = [_vp, _vp, _u64]
    lib.acg_streams_positions.argtypes = [_vp, _vp]
    lib.acg_streams_feed.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _vp, _u64, C.POINTER(_u64)]
    lib.acg_streams_feed_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _vp, _u64, _vp, C.POINTER(_u64)]
    lib.acg_streams_create_replace.argtypes = [_vp, _u64, _vp, _vp, _u64, C.POINTER(_vp)]
    lib.acg_streams_replace_feed.argtypes = [_vp, _vp, _i, _u64, _vp, _u64, _vp, _u64, _vp, C.POINTER(_u64)]
    lib.acg_streams_replace_feed_devout.argtypes = [_vp, _vp, _u64, _vp, _i, _u64, _vp, _u64, _vp,
                                                    C.POINTER(_u64)]
    lib.acg_streams_flush.argtypes = [_vp, _vp, _u64, _vp, _u64, _vp, C.POINTER(_u64)]
    lib.acg_streams_held.argtypes = [_vp, _vp]
    lib.acg_candidates_create.argtypes = [_vp, _vp, _vp, _u64, C.POINTER(_vp)]
    lib.acg_candidates_free.argtypes = [_vp]
    lib.acg_candidates_free.restype = None
    lib.acg_streams_lookahead.argtypes = [_vp, _vp, _vp, _u64, _vp]
    lib.acg_streams_lookahead_devout.argtypes = [_vp, _vp, _vp, _u64, _vp]
    lib.acg_device_count.argtypes = []
    # multi-GPU (include/acb200.h, SURVEY.md section 8e)
    lib.acg_comm_unique_id.argtypes = [_vp]
    lib.acg_comm_init.argtypes = [_vp, _i, _i, C.POINTER(_vp)]
    lib.acg_comm_free.argtypes = [_vp]
    lib.acg_comm_free.restype = None
    lib.acg_comm_rank.argtypes = [_vp]
    lib.acg_comm_size.argtypes = [_vp]
    lib.acg_comm_transport.argtypes = [_vp]
    lib.acg_shard_plan.argtypes = [_u64, _u64, _i, _i, _u64, C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]
    lib.acg_find_overlapping_sharded.argtypes = [_vp, _vp, _vp, _i, _u64, _u64, _u64, _u64, C.POINTER(_vp),
                                                  C.POINTER(_u64), _vp, _u64, _vp]
    lib.acg_find_overlapping_sharded_begin.argtypes = [_vp, _vp, _vp, _i, _u64, _u64, _u64, _u64, C.POINTER(_i)]
    lib.acg_find_overlapping_sharded_wait.argtypes = [_vp, _i, C.POINTER(_vp), C.POINTER(_u64), _vp, _u64, _vp]
    lib.acg_comm_mark.argtypes = [_vp, _i]
    lib.acg_comm_mark_elapsed_ms.argtypes = [_vp, C.POINTER(C.c_float)]
    lib.acg_comm_fetch.argtypes = [_vp, _vp, _u64, C.POINTER(_u64)]
    lib.acg_comm_fetch_view.argtypes = [_vp, C.POINTER(_vp), C.POINTER(_u64)]
    lib.acg_comm_checksum.argtypes = [_vp, C.POINTER(_u64), C.POINTER(_u64)]


_declare(_lib)


def device_count() -> int:
    return _lib.acg_device_count()


class Match:
    """`Match`, src/util/search.rs:825-830."""
    __slots__ = ("_pid", "_start", "_end")

    def __init__(self, pid, start, end):
        self._pid, self._start, self._end = int(pid), int(start), int(end)

    def pattern(self):
        return self._pid

    def start(self):
        return self._start

    def end(self):
        return self._end

    def span(self):
        return (self._start, self._end)

    def is_empty(self):
        return self._start == self._end

    def as_tuple(self):
        return (self._pid, self._start, self._end)

    def __eq__(self, o):
        return isinstance(o, Match) and self.as_tuple() == o.as_tuple()

    def __repr__(self):
        return f"Match(pattern={self._pid}, span={self._start}..{self._end})"


def _hay_ptr(hay):
    """(keepalive, address, length) of a bytes-like / contiguous uint8 ndarray haystack."""
    if isinstance(hay, np.ndarray):
        if hay.dtype != np.uint8 or not hay.flags["C_CONTIGUOUS"]:
            raise TypeError("haystack ndarray must be contiguous uint8")
        return hay, hay.ctypes.data, hay.size
    if isinstance(hay, str):
        hay = hay.encode()
    arr = np.frombuffer(bytes(hay) if not isinstance(hay, (bytes, bytearray, memoryview)) else hay, dtype=np.uint8)
    return arr, arr.ctypes.data if arr.size else 0, arr.size


def _host_offsets(offsets):
    """[n_docs + 1] CSR bounds in host memory as a uint64 ndarray."""
    offs = np.ascontiguousarray(offsets, dtype=np.int64)
    if offs.ndim != 1 or offs.size == 0 or (offs < 0).any():
        raise ValueError("document offsets must be a non-empty 1-D array of non-negative integers")
    return offs.astype(np.uint64)


def _batch_input(docs):
    """(keepalive, address, length, on_device, uint64 offsets) of a batch of documents: a list of
    bytes / str, or a (values, offsets) pair -- values a contiguous uint8 ndarray or a CUDA torch.uint8
    tensor, offsets the [n_docs + 1] CSR bounds (host, int64)."""
    if isinstance(docs, tuple) and len(docs) == 2:
        values, offsets = docs
        offs = _host_offsets(offsets)
        if getattr(values, "is_cuda", False):
            if str(values.dtype) != "torch.uint8" or not values.is_contiguous():
                raise TypeError("device haystack must be a contiguous torch.uint8 tensor")
            return values, values.data_ptr(), values.numel(), 1, offs
        keep, ptr, n = _hay_ptr(values)
        return keep, ptr, n, 0, offs
    pieces = [d.encode() if isinstance(d, str) else bytes(d) for d in docs]
    offs = np.zeros(len(pieces) + 1, dtype=np.uint64)
    if pieces:
        np.cumsum(np.fromiter(map(len, pieces), dtype=np.uint64, count=len(pieces)), out=offs[1:])
    keep, ptr, n = _hay_ptr(b"".join(pieces))
    return keep, ptr, n, 0, offs


def _devout_offsets(offsets, n_docs):
    """(keepalive, address, n_docs, on_device) of the offsets of a raw-pointer devout call: a host array of
    [n_docs + 1] bounds, or an int device address of them with n_docs given."""
    if isinstance(offsets, int):
        if n_docs is None:
            raise TypeError("offsets given as a device address need n_docs")
        return None, offsets, int(n_docs), 1
    offs = _host_offsets(offsets)
    return offs, offs.ctypes.data, offs.size - 1, 0


def _torch_batch(docs):
    """(values, offsets keepalive, offsets address, n_docs, on_device) of a (CUDA torch.uint8 values, offsets)
    batch, offsets an int64 CUDA tensor on the values' device or a host array.  Torch's current stream is
    synchronised first: the library runs on its own streams and the inputs may still be in flight."""
    import torch
    values, offsets = docs
    if not getattr(values, "is_cuda", False) or values.dtype != torch.uint8 or not values.is_contiguous():
        raise TypeError("values must be a contiguous CUDA torch.uint8 tensor")
    if isinstance(offsets, torch.Tensor) and offsets.is_cuda:
        if offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() == 0:
            raise ValueError("device document offsets must be a non-empty 1-D int64 tensor")
        if offsets.device != values.device:
            raise ValueError("document offsets must be on the haystack's device")
        offsets = offsets.contiguous()
        keep, ptr, n_docs, on_dev = offsets, offsets.data_ptr(), offsets.numel() - 1, 1
    else:
        keep, ptr, n_docs, on_dev = _devout_offsets(offsets, None)
    torch.cuda.current_stream(values.device).synchronize()
    return values, keep, ptr, n_docs, on_dev


# Device-resident batch records (find_iter_batch_torch / find_overlapping_iter_batch_torch), CUDA tensors on the
# haystack's device: `records` int64 [n, 3], the acg_doc_match words (pid | doc << 32, start, end); `offsets` int64
# [n_docs + 1], the records of document d are records[offsets[d]:offsets[d + 1]]; `pid`, `doc` [n] derived from
# records[:, 0], `start`, `end` views of its other columns.
BatchMatches = collections.namedtuple("BatchMatches", "records offsets pid doc start end")


def _span(span, n):
    if span is None:
        return 0, n
    return int(span[0]), int(span[1])


class Input:
    """`Input`, src/util/search.rs:60-720: a haystack with a span, an anchored mode and the
    `earliest` flag.  Every search method accepts either a plain haystack (with keyword arguments)
    or an `Input`."""
    __slots__ = ("_hay", "_n", "_start", "_end", "_anchored", "_earliest")

    def __init__(self, haystack):  # Input::new, :93
        keep, _, n = _hay_ptr(haystack)
        self._hay, self._n = keep, n
        self._start, self._end = 0, n
        self._anchored, self._earliest = Anchored.No, False

    new = staticmethod(lambda haystack: Input(haystack))

    def clone(self):
        c = Input.__new__(Input)
        for k in Input.__slots__:
            setattr(c, k, getattr(self, k))
        return c

    # builder-style setters (consume and return, :142-310)
    def span(self, span):
        self.set_span(span)
        return self

    def range(self, rng):
        self.set_range(rng)
        return self

    def anchored(self, mode):
        self.set_anchored(mode)
        return self

    def earliest(self, yes):
        self.set_earliest(yes)
        return self

    # setters (:332-480)
    def set_span(self, span):
        start, end = int(span[0]), int(span[1])
        # the reference panics on an invalid span (:335-341)
        if not (0 <= start and end <= self._n and start <= end + 1):
            raise ValueError(f"invalid span ({start}, {end}) for haystack of length {self._n}")
        self._start, self._end = start, end

    def set_range(self, rng):
        if isinstance(rng, (range, slice)):
            if rng.step not in (None, 1):
                raise ValueError("ranges must have step 1")
            start = 0 if rng.start is None else rng.start
            end = self._n if rng.stop is None else rng.stop
            rng = (start, end)
        self.set_span(rng)

    def set_start(self, start):
        self.set_span((start, self._end))

    def set_end(self, end):
        self.set_span((self._start, end))

    def set_anchored(self, mode):
        self._anchored = Anchored(mode)

    def set_earliest(self, yes):
        self._earliest = bool(yes)

    # getters (:493-630)
    def haystack(self):
        return self._hay

    def start(self):
        return self._start

    def end(self):
        return self._end

    def get_span(self):
        return (self._start, self._end)

    def get_range(self):
        return range(self._start, self._end)

    def get_anchored(self):
        return self._anchored

    def get_earliest(self):
        return self._earliest

    def is_done(self):  # :627
        return self._start > self._end


class OverlappingState:
    """`OverlappingState`, src/automaton.rs:782-840: the cursor of a resumable overlapping search.
    The device scan is eager, so the state holds the ordered match list of the search it was first
    used with and hands out one match per `try_find_overlapping` call -- the same sequence the
    reference's state machine produces.  As in the reference, a state must be reused only with the
    same automaton and input."""
    __slots__ = ("_matches", "_next", "_mat")

    def __init__(self):
        self._matches = None
        self._next = 0
        self._mat = None

    @staticmethod
    def start():  # :817
        return OverlappingState()

    def get_match(self):  # :829
        return self._mat


class AhoCorasickBuilder:
    """`AhoCorasickBuilder`, src/ahocorasick.rs:2135-2617 (same knobs, same defaults)."""

    def __init__(self):
        self._o = dict(match_kind=MatchKind.Standard, start_kind=StartKind.Unanchored,
                       ascii_case_insensitive=False, byte_classes=True, prefilter=True, kind=None,
                       dense_depth=3)
        self._host_only = False
        self._device_fill = False

    def match_kind(self, kind):
        self._o["match_kind"] = MatchKind(kind)
        return self

    def start_kind(self, kind):
        self._o["start_kind"] = StartKind(kind)
        return self

    def ascii_case_insensitive(self, yes):
        self._o["ascii_case_insensitive"] = bool(yes)
        return self

    def kind(self, kind):
        self._o["kind"] = None if kind is None else AhoCorasickKind(kind)
        return self

    def prefilter(self, yes):
        self._o["prefilter"] = bool(yes)
        return self

    def dense_depth(self, depth):
        self._o["dense_depth"] = int(depth)
        return self

    def byte_classes(self, yes):
        self._o["byte_classes"] = bool(yes)
        return self

    def host_only(self, yes=True):
        """Build the tables without touching CUDA (table-parity checks on CPU-only machines)."""
        self._host_only = bool(yes)
        return self

    def device_fill(self, yes=True):
        """Produce the dense transition table on the GPU (acg_build_on_device) instead of building it on
        the host and copying it over; same table, same results."""
        self._device_fill = bool(yes)
        return self

    def build(self, patterns):
        pats = [p.encode() if isinstance(p, str) else bytes(p) for p in patterns]
        n = len(pats)
        # one contiguous buffer + a pointer per pattern (a ctypes object per pattern costs ~3 us each:
        # a third of a second for the 100 000 patterns of BASELINE config 5)
        lens_np = np.fromiter((len(p) for p in pats), dtype=np.uint64, count=n) if n else np.zeros(1, np.uint64)
        blob = np.frombuffer(b"".join(pats) + b"\0", dtype=np.uint8)
        offs = np.zeros(max(n, 1), dtype=np.uint64)
        if n > 1:
            np.cumsum(lens_np[:-1], out=offs[1:n])
        ptrs = (offs + np.uint64(blob.ctypes.data)).astype(np.uint64)
        arr = ptrs.ctypes.data_as(C.POINTER(C.c_char_p))
        lens = lens_np.ctypes.data_as(C.POINTER(_u64))
        keep = (blob, ptrs, lens_np)
        o = self._o
        opts = _BuildOpts(int(o["match_kind"]), int(o["start_kind"]), int(o["ascii_case_insensitive"]),
                          int(o["byte_classes"]), int(o["prefilter"]), int(o["kind"] or 0), o["dense_depth"])
        h = _vp()
        fn = _lib.acg_build_host if self._host_only else (_lib.acg_build_on_device if self._device_fill else _lib.acg_build)
        rc = fn(arr, lens, n, C.byref(opts), C.byref(h))
        if rc in (-1, -2, -3):
            raise BuildError(rc)
        if rc:
            raise DeviceError(rc)
        return AhoCorasick(h)


def _until_it_fits(owner, cap, alloc, cnt, call):
    """The caller's side of the two-call overflow protocol: `call(out, cap)` on `out = alloc(cap)`, again with
    room to spare while it returns E_OVERFLOW (the call leaves the required count in `cnt`); `owner` keeps
    the capacity that was needed as a hint for its next search.  Returns out[:count]."""
    while True:
        out = alloc(cap)
        rc = call(out, cap)
        if rc == E_OVERFLOW:
            cap = int(cnt.value) + int(cnt.value) // 8 + 64
            owner._cap_hint = max(owner._cap_hint, cap)
            continue
        if rc:
            owner._raise(rc)
        return out[: cnt.value]


class AhoCorasick:
    """`AhoCorasick`, src/ahocorasick.rs:177-2082 (search surface only; replace/stream are out of scope)."""

    def __init__(self, handle):
        self._h = handle
        self._cap_hint = 4096  # output-buffer sizing for the two-call overflow protocol
        self._replace_ratio = 1.0  # replace_all_batch*: output bytes per input byte that a retry had to make room for

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            try:
                _lib.acg_dfa_free(h)
            except Exception:
                pass
            self._h = None

    @staticmethod
    def new(patterns):  # src/ahocorasick.rs:243
        return AhoCorasickBuilder().build(patterns)

    @staticmethod
    def builder():  # src/ahocorasick.rs:268
        return AhoCorasickBuilder()

    @staticmethod
    def from_dfa_tables(t: dict):
        """Adopt a DFA built elsewhere (what a Rust -sys shim does): acg_dfa_create."""
        d = _Desc()
        keep = {}

        def arr(name, dtype=np.uint32):
            a = np.ascontiguousarray(t[name], dtype=dtype)
            keep[name] = a
            return a.ctypes.data_as(C.POINTER(C.c_uint32))
        d.trans = arr("trans")
        d.trans_len = keep["trans"].size
        d.stride2, d.alphabet_len = int(t["stride2"]), int(t["alphabet_len"])
        bc = np.ascontiguousarray(t["byte_classes"], dtype=np.uint8)
        C.memmove(d.byte_classes, bc.ctypes.data, 256)
        for k in ("max_special_id", "max_match_id", "start_unanchored_id", "start_anchored_id"):
            setattr(d, k, int(t[k]))
        d.match_offsets = arr("match_offsets")
        d.match_pids = arr("match_pids")
        d.pattern_lens = arr("pattern_lens")
        d.n_patterns = keep["pattern_lens"].size
        d.match_kind = int(t["match_kind"])
        d.start_kind = int(t.get("start_kind", 0))
        d.prefilter_kind = int(t.get("prefilter_kind", 0))
        d.min_pattern_len, d.max_pattern_len = int(t["min_pattern_len"]), int(t["max_pattern_len"])
        h = _vp()
        rc = _lib.acg_dfa_create(C.byref(d), C.byref(h))
        if rc:
            raise DeviceError(rc)
        return AhoCorasick(h)

    # ---- getters (src/ahocorasick.rs:1867-2021) ----
    def kind(self):
        return AhoCorasickKind(_lib.acg_kind(self._h))

    def start_kind(self):
        return StartKind(_lib.acg_start_kind(self._h))

    def match_kind(self):
        return MatchKind(_lib.acg_match_kind(self._h))

    def min_pattern_len(self):
        return _lib.acg_min_pattern_len(self._h)

    def max_pattern_len(self):
        return _lib.acg_max_pattern_len(self._h)

    def patterns_len(self):
        return _lib.acg_patterns_len(self._h)

    def memory_usage(self):
        return _lib.acg_memory_usage(self._h)

    def prefilter_kind(self):
        return _lib.acg_prefilter_kind(self._h)

    def packed_variant(self):
        fat, ml = _i(), _i()
        if not _lib.acg_packed_variant(self._h, C.byref(fat), C.byref(ml)):
            return None
        return {"fat": bool(fat.value), "mask_len": ml.value}

    def state_len(self):
        return _lib.acg_dfa_state_len(self._h)

    def tables(self) -> dict:
        d = _Desc()
        rc = _lib.acg_dfa_table(self._h, C.byref(d))  # fetches the table of a device-filled handle
        if rc:
            raise DeviceError(rc)
        nms = (d.max_match_id >> d.stride2) - 1

        def arr(ptr, n):
            return np.ctypeslib.as_array(ptr, (n,)).copy() if n and ptr else np.zeros(0, np.uint32)
        offs = arr(d.match_offsets, nms + 1)
        tot = int(offs[-1])
        return {
            "trans": arr(d.trans, d.trans_len),
            "stride2": d.stride2, "alphabet_len": d.alphabet_len,
            "byte_classes": np.frombuffer(bytes(d.byte_classes), dtype=np.uint8).copy(),
            "max_special_id": d.max_special_id, "max_match_id": d.max_match_id,
            "start_unanchored_id": d.start_unanchored_id, "start_anchored_id": d.start_anchored_id,
            "match_offsets": offs,
            "match_pids": arr(d.match_pids, tot),
            "pattern_lens": arr(d.pattern_lens, d.n_patterns),
            "match_kind": d.match_kind, "start_kind": d.start_kind, "prefilter_kind": d.prefilter_kind,
            "min_pattern_len": d.min_pattern_len, "max_pattern_len": d.max_pattern_len,
            "state_len": _lib.acg_dfa_state_len(self._h),
        }

    # ---- engine control / stats (device-side knobs that do not exist in the reference) ----
    def set_engine(self, engine):
        rc = _lib.acg_set_engine(self._h, int(engine))
        if rc:
            raise DeviceError(rc)
        return self

    def last_stats(self) -> dict:
        s = _Stats()
        _lib.acg_last_stats(self._h, C.byref(s))
        return {k: getattr(s, k) for k, _ in _Stats._fields_}

    # ---- searches ----
    @staticmethod
    def _raise(rc):
        if -14 <= rc <= -10:
            raise MatchError(rc)
        if rc == -20:
            raise ValueError("invalid span for haystack")  # the reference panics (search.rs:332-343)
        raise DeviceError(rc)

    def _collect(self, fn, hay, span, anchored):
        if isinstance(hay, Input):
            hay, span, anchored = hay.haystack(), hay.get_span(), hay.get_anchored()
        keep, ptr, n = _hay_ptr(hay)
        s, e = _span(span, n)
        # room for one match per 256 haystack bytes from the start (the device sizes its own tuple buffer the
        # same way): an overflow retry repeats the whole copy + scan, so it should be the exception
        cnt = _u64()
        return _until_it_fits(
            self, max(self._cap_hint, max(e - s, 0) // 256 + 64), lambda cap: np.empty(cap, MATCH_DTYPE), cnt,
            lambda out, cap: fn(self._h, ptr, n, s, e, int(anchored), out.ctypes.data, cap, C.byref(cnt)))

    def try_find_iter_np(self, hay, span=None, anchored=Anchored.No):
        return self._collect(_lib.acg_find_iter, hay, span, anchored)

    def try_find_overlapping_iter_np(self, hay, span=None, anchored=Anchored.No):
        return self._collect(_lib.acg_find_overlapping, hay, span, anchored)

    def try_find_iter(self, hay, span=None, anchored=Anchored.No):  # src/ahocorasick.rs:1275
        r = self.try_find_iter_np(hay, span, anchored)
        return [Match(a, b, c) for a, b, c in zip(r["pid"], r["start"], r["end"])]

    def try_find_overlapping_iter(self, hay, span=None, anchored=Anchored.No):  # :1350
        r = self.try_find_overlapping_iter_np(hay, span, anchored)
        return [Match(a, b, c) for a, b, c in zip(r["pid"], r["start"], r["end"])]

    def try_find_overlapping(self, hay, state: OverlappingState, span=None, anchored=Anchored.No):
        """`try_find_overlapping`, src/ahocorasick.rs:1184: advance `state` to the next overlapping
        match (or to None).  Errors are the ones of try_find_overlapping_iter (src/automaton.rs
        :397-423) and are reported on every call, as in the reference."""
        if state._matches is None:
            state._matches = self.try_find_overlapping_iter(hay, span, anchored)
            state._next = 0
        if state._next < len(state._matches):
            state._mat = state._matches[state._next]
            state._next += 1
        else:
            state._mat = None

    find_overlapping = try_find_overlapping  # :470

    find_iter = try_find_iter  # :562 (the infallible versions panic where these raise)
    find_overlapping_iter = try_find_overlapping_iter  # :609

    def try_find(self, hay, span=None, anchored=Anchored.No, earliest=False):  # :1021
        if isinstance(hay, Input):
            hay, span, anchored, earliest = hay.haystack(), hay.get_span(), hay.get_anchored(), hay.get_earliest()
        keep, ptr, n = _hay_ptr(hay)
        s, e = _span(span, n)
        out = np.zeros(1, MATCH_DTYPE)
        found = _i()
        rc = _lib.acg_find(self._h, ptr, n, s, e, int(anchored), int(earliest), out.ctypes.data, C.byref(found))
        if rc:
            self._raise(rc)
        if not found.value:
            return None
        return Match(out["pid"][0], out["start"][0], out["end"][0])

    find = try_find  # :404

    def is_match(self, hay, span=None):  # :311
        # The reference asks for the earliest match; only existence is reported, and a match exists
        # under `earliest` iff one exists without it, so leftmost automata stay on the windowed
        # device scan instead of the single-lane engine.
        earliest = self.match_kind() == MatchKind.Standard
        if isinstance(hay, Input):
            return self.try_find(hay.clone().earliest(earliest)) is not None
        return self.try_find(hay, span, earliest=earliest) is not None

    # ---- batched search: many documents in one device call (include/acb200.h, acg_*_batch) ----
    # `docs`: a list of bytes / str, or (values, offsets) with values a uint8 ndarray or a CUDA
    # torch.uint8 tensor and offsets the host int64 CSR bounds [n_docs + 1].  Per document the results are
    # those of the single-haystack call on that document alone, offsets relative to it.
    def _collect_batch(self, fn, docs, anchored):
        keep, ptr, n, on_dev, offs = _batch_input(docs)
        n_docs = offs.size - 1
        cnt = _u64()
        out = _until_it_fits(
            self, max(self._cap_hint, n // 256 + 64), lambda cap: np.empty(cap, DOC_MATCH_DTYPE), cnt,
            lambda out, cap: fn(self._h, ptr, on_dev, n, offs.ctypes.data, n_docs, int(anchored), out.ctypes.data,
                                cap, C.byref(cnt)))
        return out, n_docs

    @staticmethod
    def _per_doc(r, n_docs):
        res = [[] for _ in range(n_docs)]
        for d, p, s, e in zip(r["doc"].tolist(), r["pid"].tolist(), r["start"].tolist(), r["end"].tolist()):
            res[d].append(Match(p, s, e))
        return res

    def find_iter_batch_np(self, docs, anchored=Anchored.No):
        """find_iter of every document: structured array (doc, pid, start, end), ascending doc."""
        return self._collect_batch(_lib.acg_find_iter_batch, docs, anchored)[0]

    def find_overlapping_iter_batch_np(self, docs, anchored=Anchored.No):
        return self._collect_batch(_lib.acg_find_overlapping_batch, docs, anchored)[0]

    def find_iter_batch(self, docs, anchored=Anchored.No):
        """find_iter of every document: one list of Match per document."""
        return self._per_doc(*self._collect_batch(_lib.acg_find_iter_batch, docs, anchored))

    def find_overlapping_iter_batch(self, docs, anchored=Anchored.No):
        return self._per_doc(*self._collect_batch(_lib.acg_find_overlapping_batch, docs, anchored))

    def is_match_batch(self, docs, anchored=Anchored.No):
        """is_match of every document: bool array [n_docs]."""
        keep, ptr, n, on_dev, offs = _batch_input(docs)
        flags = np.zeros(max(offs.size - 1, 1), dtype=np.uint8)
        rc = _lib.acg_is_match_batch(self._h, ptr, on_dev, n, offs.ctypes.data, offs.size - 1, int(anchored),
                                     flags.ctypes.data)
        if rc:
            self._raise(rc)
        return flags[: offs.size - 1].astype(bool)

    def find_batch_np(self, docs, anchored=Anchored.No, earliest=False):
        """try_find of every document: (found, bool [n_docs]; records, DOC_MATCH_DTYPE [n_docs]).  A document
        without a match has found False and the record (pid 0, doc, 0, 0)."""
        keep, ptr, n, on_dev, offs = _batch_input(docs)
        n_docs = offs.size - 1
        found = np.empty(max(n_docs, 1), dtype=np.uint8)
        out = np.empty(max(n_docs, 1), DOC_MATCH_DTYPE)
        rc = _lib.acg_find_batch(self._h, ptr, on_dev, n, offs.ctypes.data, n_docs, int(anchored), int(earliest),
                                 out.ctypes.data, found.ctypes.data)
        if rc:
            self._raise(rc)
        return found[:n_docs].astype(bool), out[:n_docs]

    def find_batch(self, docs, anchored=Anchored.No, earliest=False):
        """try_find of every document: one Match, or None, per document."""
        found, r = self.find_batch_np(docs, anchored, earliest)
        return [Match(p, s, e) if f else None
                for f, p, s, e in zip(found.tolist(), r["pid"].tolist(), r["start"].tolist(), r["end"].tolist())]

    # ---- batched search with device-resident results (acg_*_batch_devout) ----
    # Raw-pointer forms: d_hay_ptr / out_ptr / match_offsets_ptr / flags_ptr / found_ptr are device addresses;
    # `offsets` is a host array of [n_docs + 1] bounds, or an int device address of them with `n_docs` given.
    def _batch_devout(self, fn, d_hay_ptr, hay_len, offsets, out_ptr, cap, match_offsets_ptr, anchored, n_docs):
        keep, optr, n_docs, on_dev = _devout_offsets(offsets, n_docs)
        cnt = _u64()
        rc = fn(self._h, d_hay_ptr, hay_len, optr, on_dev, n_docs, int(anchored), out_ptr, cap, match_offsets_ptr,
                C.byref(cnt))
        if rc == E_OVERFLOW:
            raise OverflowError(int(cnt.value))
        if rc:
            self._raise(rc)
        return int(cnt.value)

    def find_iter_batch_devout(self, d_hay_ptr, hay_len, offsets, out_ptr, cap, match_offsets_ptr,
                               anchored=Anchored.No, n_docs=None):
        """find_iter of every document into device memory: acg_doc_match records at out_ptr and their CSR index
        by document ([n_docs + 1] uint64) at match_offsets_ptr.  Returns the record count; raises
        OverflowError(needed) if cap is too small (nothing is written then)."""
        return self._batch_devout(_lib.acg_find_iter_batch_devout, d_hay_ptr, hay_len, offsets, out_ptr, cap,
                                  match_offsets_ptr, anchored, n_docs)

    def find_overlapping_iter_batch_devout(self, d_hay_ptr, hay_len, offsets, out_ptr, cap, match_offsets_ptr,
                                           anchored=Anchored.No, n_docs=None):
        return self._batch_devout(_lib.acg_find_overlapping_batch_devout, d_hay_ptr, hay_len, offsets, out_ptr, cap,
                                  match_offsets_ptr, anchored, n_docs)

    def is_match_batch_devout(self, d_hay_ptr, hay_len, offsets, flags_ptr, anchored=Anchored.No, n_docs=None):
        """is_match of every document: flags_ptr[d] = 0 / 1 (uint8, device)."""
        keep, optr, n_docs, on_dev = _devout_offsets(offsets, n_docs)
        rc = _lib.acg_is_match_batch_devout(self._h, d_hay_ptr, hay_len, optr, on_dev, n_docs, int(anchored),
                                            flags_ptr)
        if rc:
            self._raise(rc)

    def find_batch_devout(self, d_hay_ptr, hay_len, offsets, out_ptr, found_ptr, anchored=Anchored.No,
                          earliest=False, n_docs=None):
        """try_find of every document: found_ptr[d] (uint8) and the record out_ptr[d] (acg_doc_match), device."""
        keep, optr, n_docs, on_dev = _devout_offsets(offsets, n_docs)
        rc = _lib.acg_find_batch_devout(self._h, d_hay_ptr, hay_len, optr, on_dev, n_docs, int(anchored),
                                        int(earliest), out_ptr, found_ptr)
        if rc:
            self._raise(rc)

    # Torch forms: `docs` = (values, offsets), values a CUDA torch.uint8 tensor, offsets an int64 CUDA tensor on
    # its device or a host array; the results are CUDA tensors on the values' device.
    def _collect_batch_torch(self, fn, docs, anchored):
        import torch
        values, keep, optr, n_docs, on_dev = _torch_batch(docs)
        match_offsets = torch.empty(n_docs + 1, dtype=torch.int64, device=values.device)
        cnt = _u64()
        r = _until_it_fits(
            self, self._cap_hint, lambda cap: torch.empty((cap, 3), dtype=torch.int64, device=values.device), cnt,
            lambda records, cap: fn(self._h, values.data_ptr(), values.numel(), optr, on_dev, n_docs, int(anchored),
                                    records.data_ptr(), cap, match_offsets.data_ptr(), C.byref(cnt)))
        return BatchMatches(r, match_offsets, r[:, 0] & 0xFFFFFFFF, r[:, 0] >> 32, r[:, 1], r[:, 2])

    def find_iter_batch_torch(self, docs, anchored=Anchored.No):
        """find_iter of every document, results on the device: a BatchMatches of CUDA tensors."""
        return self._collect_batch_torch(_lib.acg_find_iter_batch_devout, docs, anchored)

    def find_overlapping_iter_batch_torch(self, docs):
        return self._collect_batch_torch(_lib.acg_find_overlapping_batch_devout, docs, Anchored.No)

    def is_match_batch_torch(self, docs, anchored=Anchored.No):
        """is_match of every document: CUDA bool tensor [n_docs]."""
        import torch
        values, keep, optr, n_docs, on_dev = _torch_batch(docs)
        flags = torch.empty(n_docs, dtype=torch.bool, device=values.device)
        rc = _lib.acg_is_match_batch_devout(self._h, values.data_ptr(), values.numel(), optr, on_dev, n_docs,
                                            int(anchored), flags.data_ptr())
        if rc:
            self._raise(rc)
        return flags

    def find_batch_torch(self, docs, anchored=Anchored.No, earliest=False):
        """try_find of every document: (found, CUDA bool [n_docs]; records, CUDA int64 [n_docs, 3] acg_doc_match
        words).  A document without a match has found False and the record (0 | doc << 32, 0, 0)."""
        import torch
        values, keep, optr, n_docs, on_dev = _torch_batch(docs)
        found = torch.empty(n_docs, dtype=torch.bool, device=values.device)
        records = torch.empty((n_docs, 3), dtype=torch.int64, device=values.device)
        rc = _lib.acg_find_batch_devout(self._h, values.data_ptr(), values.numel(), optr, on_dev, n_docs,
                                        int(anchored), int(earliest), records.data_ptr(), found.data_ptr())
        if rc:
            self._raise(rc)
        return found, records

    # ---- pattern counts per document (acg_pattern_counts_batch) ----
    # How often each pattern occurs in each document: the records of find_overlapping_iter_batch (overlapping) or
    # find_iter_batch, counted by (document, pattern) on the device, as a CSR matrix [n_docs x patterns_len()].
    def _counts_until_it_fits(self, alloc, call):
        """The two-call overflow protocol for the (pids, counts) arrays: returns (pids, counts) cut to nnz."""
        cnt = _u64()
        cap = self._cap_hint
        while True:
            pids, counts = alloc(cap)
            rc = call(pids, counts, cap, C.byref(cnt))
            if rc == E_OVERFLOW:
                cap = int(cnt.value) + int(cnt.value) // 8 + 64
                self._cap_hint = max(self._cap_hint, cap)
                continue
            if rc:
                self._raise(rc)
            return pids[: cnt.value], counts[: cnt.value]

    def pattern_counts_batch_np(self, docs, overlapping=False, anchored=Anchored.No):
        """(row_offsets uint64 [n_docs + 1], pids uint32 [nnz], counts uint64 [nnz]): document d's patterns are
        pids[row_offsets[d]:row_offsets[d + 1]], ascending, each occurring counts[i] times in it.  `docs` as in
        find_iter_batch_np."""
        keep, ptr, n, on_dev, offs = _batch_input(docs)
        n_docs = offs.size - 1
        rows = np.empty(n_docs + 1, dtype=np.uint64)
        pids, counts = self._counts_until_it_fits(
            lambda cap: (np.empty(cap, np.uint32), np.empty(cap, np.uint64)),
            lambda pids, counts, cap, nnz: _lib.acg_pattern_counts_batch(
                self._h, ptr, on_dev, n, offs.ctypes.data, n_docs, int(anchored), int(overlapping), rows.ctypes.data,
                pids.ctypes.data, counts.ctypes.data, cap, nnz))
        return rows, pids, counts

    def pattern_counts_batch_devout(self, d_hay_ptr, hay_len, offsets, row_offsets_ptr, pids_ptr, counts_ptr, cap,
                                    overlapping=False, anchored=Anchored.No, n_docs=None):
        """The counts into device memory: row_offsets_ptr [n_docs + 1] uint64, pids_ptr [cap] uint32, counts_ptr
        [cap] uint64.  Returns nnz; raises OverflowError(needed) if cap is too small (nothing is written then)."""
        keep, optr, n_docs, on_dev = _devout_offsets(offsets, n_docs)
        nnz = _u64()
        rc = _lib.acg_pattern_counts_batch_devout(self._h, d_hay_ptr, hay_len, optr, on_dev, n_docs, int(anchored),
                                                  int(overlapping), row_offsets_ptr, pids_ptr, counts_ptr, cap,
                                                  C.byref(nnz))
        if rc == E_OVERFLOW:
            raise OverflowError(int(nnz.value))
        if rc:
            self._raise(rc)
        return int(nnz.value)

    def pattern_counts_batch_torch(self, docs, overlapping=False, anchored=Anchored.No):
        """The counts as a CUDA torch.sparse_csr_tensor of size (n_docs, patterns_len()) on the values' device, with
        int64 crow / col indices and values.  `docs` as in find_iter_batch_torch."""
        import torch
        values, keep, optr, n_docs, on_dev = _torch_batch(docs)
        dev = values.device
        rows = torch.empty(n_docs + 1, dtype=torch.int64, device=dev)
        pids, counts = self._counts_until_it_fits(
            lambda cap: (torch.empty(cap, dtype=torch.int32, device=dev), torch.empty(cap, dtype=torch.int64, device=dev)),
            lambda pids, counts, cap, nnz: _lib.acg_pattern_counts_batch_devout(
                self._h, values.data_ptr(), values.numel(), optr, on_dev, n_docs, int(anchored), int(overlapping),
                rows.data_ptr(), pids.data_ptr(), counts.data_ptr(), cap, nnz))
        return torch.sparse_csr_tensor(rows, pids.to(torch.int64), counts, size=(n_docs, self.patterns_len()))

    # ---- match coverage per document (acg_match_coverage_batch) ----
    # How much of each document the records of find_overlapping_iter_batch (overlapping) or find_iter_batch cover:
    # the bytes inside at least one match, per document, and optionally the per-byte mask, from the device.
    def match_coverage_batch_np(self, docs, overlapping=False, anchored=Anchored.No, mask=False):
        """covered, uint64 [n_docs]: the bytes of each document inside at least one of its matches (empty matches
        cover nothing).  With mask=True also a bool array the length of the values buffer, True where a byte lies
        in a match of its document (False outside [offsets[0], offsets[-1])).  `docs` as in find_iter_batch_np."""
        keep, ptr, n, on_dev, offs = _batch_input(docs)
        n_docs = offs.size - 1
        covered = np.empty(n_docs, dtype=np.uint64)
        m = np.zeros(n, dtype=np.uint8) if mask else None
        rc = _lib.acg_match_coverage_batch(self._h, ptr, on_dev, n, offs.ctypes.data, n_docs, int(anchored),
                                           int(overlapping), covered.ctypes.data, m.ctypes.data if mask else None)
        if rc:
            self._raise(rc)
        return (covered, m.view(bool)) if mask else covered

    def match_coverage_batch_devout(self, d_hay_ptr, hay_len, offsets, covered_ptr, mask_ptr=None, overlapping=False,
                                    anchored=Anchored.No, n_docs=None):
        """The coverage into device memory: covered_ptr [n_docs] uint64 and, unless mask_ptr is None, the mask
        (uint8, indexed like the haystack: only [offsets[0], offsets[n_docs]) is written)."""
        keep, optr, n_docs, on_dev = _devout_offsets(offsets, n_docs)
        rc = _lib.acg_match_coverage_batch_devout(self._h, d_hay_ptr, hay_len, optr, on_dev, n_docs, int(anchored),
                                                  int(overlapping), covered_ptr, mask_ptr)
        if rc:
            self._raise(rc)

    def match_coverage_batch_torch(self, docs, overlapping=False, anchored=Anchored.No, mask=True):
        """(covered, CUDA int64 [n_docs]; mask, CUDA bool [values.numel()] or None) on the values' device.  The
        mask is False outside [offsets[0], offsets[-1]).  `docs` as in find_iter_batch_torch."""
        import torch
        values, keep, optr, n_docs, on_dev = _torch_batch(docs)
        covered = torch.empty(n_docs, dtype=torch.int64, device=values.device)
        m = torch.zeros(values.numel(), dtype=torch.bool, device=values.device) if mask else None
        if mask:
            torch.cuda.current_stream(values.device).synchronize()  # the zeros are written before the call's own
        rc = _lib.acg_match_coverage_batch_devout(self._h, values.data_ptr(), values.numel(), optr, on_dev, n_docs,
                                                  int(anchored), int(overlapping), covered.data_ptr(),
                                                  m.data_ptr() if mask else None)
        if rc:
            self._raise(rc)
        return covered, m

    # ---- replace per document (acg_replace_all_batch) ----
    # replace_all_bytes of every document in one device call: the documents of a batch with the matches of
    # find_iter_batch replaced by their patterns' replacements, spliced on the device.  The result is a batch in
    # the (values, offsets) form the batch calls take.
    def _replacement_table(self, replace_with):
        """(keepalive, bytes address or None, uint64 offsets [patterns_len() + 1]) of the replacements; ValueError
        unless there is one per pattern."""
        reps = self._replacements(replace_with)
        offs = np.zeros(len(reps) + 1, dtype=np.uint64)
        if reps:
            np.cumsum(np.fromiter(map(len, reps), dtype=np.uint64, count=len(reps)), out=offs[1:])
        data = np.frombuffer(b"".join(reps), dtype=np.uint8)
        return data, data.ctypes.data if data.size else None, offs

    def _replace_until_it_fits(self, span, alloc, call):
        """The two-call overflow protocol in output bytes: `call(out, cap, out_len)` on `out = alloc(cap)`, the
        first guess the span plus an eighth and 4 KiB, scaled by the largest growth a retry of this handle has
        met.  Returns out[:out_len]."""
        cnt = _u64()
        cap = int(span * self._replace_ratio) + span // 8 + 4096
        while True:
            out = alloc(cap)
            rc = call(out, cap, C.byref(cnt))
            if rc == E_OVERFLOW:
                need = int(cnt.value)
                cap = need + need // 8 + 4096
                self._replace_ratio = max(self._replace_ratio, need / max(span, 1))
                continue
            if rc:
                self._raise(rc)
            return out[: cnt.value]

    def replace_all_batch_np(self, docs, replace_with):
        """(values uint8, offsets uint64 [n_docs + 1]): document d with every find_iter match replaced by
        replace_with[pattern] is values[offsets[d]:offsets[d + 1]], as replace_all_bytes(document) returns it.
        `docs` as in find_iter_batch_np; one replacement (bytes / str) per pattern."""
        keep, ptr, n, on_dev, offs = _batch_input(docs)
        n_docs = offs.size - 1
        rkeep, rptr, roffs = self._replacement_table(replace_with)
        out_offsets = np.empty(n_docs + 1, dtype=np.uint64)
        values = self._replace_until_it_fits(
            int(offs[-1]) - int(offs[0]), lambda cap: np.empty(cap, dtype=np.uint8),
            lambda out, cap, cnt: _lib.acg_replace_all_batch(
                self._h, ptr, on_dev, n, offs.ctypes.data, n_docs, rptr, roffs.ctypes.data, roffs.size - 1,
                out.ctypes.data, cap, out_offsets.ctypes.data, cnt))
        return values, out_offsets

    def replace_all_batch(self, docs, replace_with):
        """replace_all_bytes of every document: one bytes object per document."""
        values, offs = self.replace_all_batch_np(docs, replace_with)
        b, o = values.tobytes(), offs.tolist()
        return [b[o[d]:o[d + 1]] for d in range(len(o) - 1)]

    def replace_all_batch_devout(self, d_hay_ptr, hay_len, offsets, replace_with, out_ptr, cap, out_offsets_ptr,
                                 n_docs=None):
        """The replaced documents into device memory: the bytes at out_ptr (cap bytes of room) and their offsets,
        [n_docs + 1] uint64, at out_offsets_ptr.  Returns the output length; raises OverflowError(needed) if cap
        is too small (nothing is written then)."""
        keep, optr, n_docs, on_dev = _devout_offsets(offsets, n_docs)
        rkeep, rptr, roffs = self._replacement_table(replace_with)
        cnt = _u64()
        rc = _lib.acg_replace_all_batch_devout(self._h, d_hay_ptr, hay_len, optr, on_dev, n_docs, rptr,
                                               roffs.ctypes.data, roffs.size - 1, out_ptr, cap, out_offsets_ptr,
                                               C.byref(cnt))
        if rc == E_OVERFLOW:
            raise OverflowError(int(cnt.value))
        if rc:
            self._raise(rc)
        return int(cnt.value)

    def replace_all_batch_torch(self, docs, replace_with):
        """(values, CUDA uint8; offsets, CUDA int64 [n_docs + 1]) on the values' device: the replaced documents as
        a batch.  `docs` as in find_iter_batch_torch."""
        import torch
        values, keep, optr, n_docs, on_dev = _torch_batch(docs)
        dev = values.device
        rkeep, rptr, roffs = self._replacement_table(replace_with)
        span = values.numel() if on_dev else int(keep[-1]) - int(keep[0])
        out_offsets = torch.empty(n_docs + 1, dtype=torch.int64, device=dev)
        out = self._replace_until_it_fits(
            span, lambda cap: torch.empty(cap, dtype=torch.uint8, device=dev),
            lambda out, cap, cnt: _lib.acg_replace_all_batch_devout(
                self._h, values.data_ptr(), values.numel(), optr, on_dev, n_docs, rptr, roffs.ctypes.data,
                roffs.size - 1, out.data_ptr(), cap, out_offsets.data_ptr(), cnt))
        return out, out_offsets

    # ---- replace / stream: host-side glue over find_iter, as in the reference -------------------
    @staticmethod
    def _is_char_boundary(view, n, i):
        """`str::is_char_boundary` on UTF-8 bytes."""
        if i == 0 or i == n:
            return True
        return i < n and (view[i] & 0xC0) != 0x80

    @staticmethod
    def _splice(view, n, matches, dst: bytearray, replace_with, char_boundaries=False):
        """The loop of `try_replace_all_with{,_bytes}`, src/automaton.rs:498-550, over an already
        materialised match list.  With `char_boundaries` (the `&str` flavour) matches that split a
        UTF-8 code point are skipped (:514-518)."""
        last = 0
        for m in matches:
            if char_boundaries and not (AhoCorasick._is_char_boundary(view, n, m.start())
                                        and AhoCorasick._is_char_boundary(view, n, m.end())):
                continue
            dst += bytes(view[last:m.start()])
            last = m.end()
            if not replace_with(m, bytes(view[m.start():m.end()]), dst):
                break
        dst += bytes(view[last:])

    def try_replace_all_with(self, hay, dst: bytearray, replace_with):
        """`try_replace_all_with_bytes`, src/automaton.rs:525-550: `replace_with(match, matched
        bytes, dst) -> bool`; returning False stops the replacement after that match."""
        keep, ptr, n = _hay_ptr(hay)
        view = memoryview(keep).cast("B") if n else b""
        self._splice(view, n, self.try_find_iter(keep), dst, replace_with)

    def _replacements(self, replace_with):
        if len(replace_with) != self.patterns_len():
            raise ValueError("replace_all requires a replacement for every pattern in the automaton")
        return [r.encode() if isinstance(r, str) else bytes(r) for r in replace_with]

    def try_replace_all_bytes(self, hay, replace_with):  # src/automaton.rs:457-480
        reps = self._replacements(replace_with)
        dst = bytearray()

        def put(m, _, out):
            out += reps[m.pattern()]
            return True
        self.try_replace_all_with(hay, dst, put)
        return bytes(dst)

    def try_replace_all(self, hay: str, replace_with):  # src/automaton.rs:433-455 -> :498-523
        reps = self._replacements(replace_with)
        keep, ptr, n = _hay_ptr(hay.encode())
        view = memoryview(keep).cast("B") if n else b""
        dst = bytearray()

        def put(m, _, out):
            out += reps[m.pattern()]
            return True
        self._splice(view, n, self.try_find_iter(keep), dst, put, char_boundaries=True)
        return dst.decode()

    replace_all = try_replace_all                # src/ahocorasick.rs:651
    replace_all_bytes = try_replace_all_bytes    # :693
    replace_all_with = try_replace_all_with      # :834 (bytes flavour)

    def _stream_chunks(self, rdr, chunk_bytes):
        """`StreamChunkIter`, src/automaton.rs:1059-1256: the stream as an alternation of
        ("bytes", data) for text between matches and ("match", Match, matched bytes), offsets
        relative to the start of the stream.  Like the reference it is limited to
        MatchKind::Standard without empty patterns (:1087-1103), and like the reference's roll buffer
        (src/util/buffer.rs) only max_pattern_len-1 bytes are carried from one device scan to the
        next: a match that straddles a block boundary starts no earlier than that."""
        if self.match_kind() != MatchKind.Standard:
            raise MatchError(-12)
        if self.patterns_len() and self.min_pattern_len() == 0:
            raise MatchError(-14)
        back = max(self.max_pattern_len() - 1, 0)
        carry = b""
        base = 0          # stream offset of carry[0]
        cursor = 0        # stream offset where the iterator restarts
        emitted = 0       # stream offset up to which chunks have been yielded
        while True:
            block = rdr.read(chunk_bytes)
            if not block:
                break
            buf = np.frombuffer(carry + bytes(block), dtype=np.uint8)
            r = self.try_find_iter_np(buf, span=(cursor - base, buf.size))
            for pid, s, e in zip(r["pid"].tolist(), r["start"].tolist(), r["end"].tolist()):
                if base + s > emitted:
                    yield ("bytes", buf[emitted - base:s].tobytes())
                yield ("match", Match(pid, base + s, base + e), buf[s:e].tobytes())
                emitted = base + e
            if len(r):
                cursor = base + int(r["end"][-1])
            keep_from = max(cursor, base + buf.size - back)
            if keep_from > emitted:  # these bytes can no longer be part of a match
                yield ("bytes", buf[emitted - base:keep_from - base].tobytes())
                emitted = keep_from
            carry = buf[keep_from - base:].tobytes()
            base = keep_from
            cursor = max(cursor, base)
        if emitted - base < len(carry):
            yield ("bytes", carry[emitted - base:])

    def try_stream_find_iter(self, rdr, chunk_bytes=64 << 20):
        """`try_stream_find_iter`, src/ahocorasick.rs:1677: matches of a byte stream (anything with
        .read(n)); equals find_iter over the concatenated stream."""
        for chunk in self._stream_chunks(rdr, chunk_bytes):
            if chunk[0] == "match":
                yield chunk[1]

    stream_find_iter = try_stream_find_iter      # :906

    def streams(self, n_streams, overlapping=False):
        """A set of n_streams byte streams searched on the device as their bytes arrive (acg_streams_*): each
        feed returns the matches that end in the bytes it brought, with offsets into the whole stream."""
        return Streams(self, n_streams, overlapping)

    def replace_streams(self, n_streams, replace_with):
        """A set of n_streams byte streams whose text is replaced on the device as their bytes arrive
        (acg_streams_create_replace): each feed returns, per stream, the text that can no longer change, with every
        find_iter match replaced by replace_with[pattern] (the forms replace_all_batch takes).  A stream's outputs,
        followed by its flush, are replace_all_bytes of everything it received, as stream_replace_all writes it."""
        return ReplaceStreams(self, n_streams, replace_with)

    def candidates(self, cands):
        """A fixed list of candidate chunks on the device (acg_candidates_create) -- a list of bytes / str, or
        (values, offsets) as the batch calls take -- for the lookahead of this automaton's stream sets."""
        return Candidates(self, cands)

    def try_stream_replace_all_with(self, rdr, wtr, replace_with, chunk_bytes=64 << 20):
        """`try_stream_replace_all_with`, src/ahocorasick.rs:1807 -> src/automaton.rs:601-636:
        `replace_with(match, matched bytes, wtr)` writes the replacement; text between matches is
        copied through as soon as it can no longer be part of a match."""
        for chunk in self._stream_chunks(rdr, chunk_bytes):
            if chunk[0] == "bytes":
                wtr.write(chunk[1])
            else:
                replace_with(chunk[1], chunk[2], wtr)

    def try_stream_replace_all(self, rdr, wtr, replace_with, chunk_bytes=64 << 20):  # :1751
        if len(replace_with) != self.patterns_len():
            raise ValueError("stream_replace_all requires a replacement for every pattern in the automaton")
        reps = [r.encode() if isinstance(r, str) else bytes(r) for r in replace_with]
        self.try_stream_replace_all_with(rdr, wtr, lambda m, _, w: w.write(reps[m.pattern()]), chunk_bytes)

    stream_replace_all = try_stream_replace_all            # :964
    stream_replace_all_with = try_stream_replace_all_with  # :1007

    # ---- device-resident haystack (torch tensor / raw pointer), for the roofline measurement ----
    def find_overlapping_iter_dev_np(self, dev_ptr, hay_len, span=None):
        s, e = _span(span, hay_len)
        cnt, ms = _u64(), C.c_float()
        out = _until_it_fits(
            self, max(self._cap_hint, 1 << 16), lambda cap: np.empty(cap, MATCH_DTYPE), cnt,
            lambda out, cap: _lib.acg_find_overlapping_dev(self._h, dev_ptr, hay_len, s, e, out.ctypes.data, cap,
                                                           C.byref(cnt), C.byref(ms)))
        return out, ms.value

    def find_iter_dev_np(self, dev_ptr, hay_len, span=None):
        s, e = _span(span, hay_len)
        cnt, ms = _u64(), C.c_float()
        out = _until_it_fits(
            self, max(self._cap_hint, 1 << 16), lambda cap: np.empty(cap, MATCH_DTYPE), cnt,
            lambda out, cap: _lib.acg_find_iter_dev(self._h, dev_ptr, hay_len, s, e, out.ctypes.data, cap,
                                                    C.byref(cnt), C.byref(ms)))
        return out, ms.value

    def find_overlapping_devout(self, dev_ptr, hay_len, span, min_end, offset_add, out_ptr, cap):
        """Ordered matches stay on the device (acg_match records at out_ptr). Returns (n, kernel_ms);
        raises OverflowError(needed) if cap is too small."""
        s, e = _span(span, hay_len)
        cnt, ms = _u64(), C.c_float()
        rc = _lib.acg_find_overlapping_devout(self._h, dev_ptr, hay_len, s, e, min_end, offset_add,
                                              out_ptr, cap, C.byref(cnt), C.byref(ms))
        if rc == E_OVERFLOW:
            raise OverflowError(int(cnt.value))
        if rc:
            self._raise(rc)
        return int(cnt.value), ms.value

    def count_overlapping_dev(self, dev_ptr, hay_len, span=None):
        s, e = _span(span, hay_len)
        cnt, fnv, ms = _u64(), _u64(), C.c_float()
        rc = _lib.acg_count_overlapping_dev(self._h, dev_ptr, hay_len, s, e, C.byref(cnt), C.byref(fnv),
                                            C.byref(ms))
        if rc:
            self._raise(rc)
        return cnt.value, fnv.value, ms.value


class _StreamSet:
    """What every stream set (Streams, ReplaceStreams) has: handle, life cycle, reset, positions, lookahead."""

    def close(self):
        if self._h and _lib is not None:
            _lib.acg_streams_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, n_chunks):
        if not self._h:
            raise ValueError("the stream set is closed")
        if n_chunks != self.n_streams:
            raise ValueError(f"a feed takes one chunk per stream: {n_chunks} chunks for {self.n_streams} streams")

    @staticmethod
    def _ids(ids):
        """(keepalive uint64 array or None, its address or None, its length) of stream ids (None: every stream)."""
        if ids is None:
            return None, None, 0
        a = np.ascontiguousarray(np.asarray(ids, dtype=np.int64).reshape(-1))
        if (a < 0).any():
            raise ValueError("stream ids must be non-negative")
        a = a.astype(np.uint64)
        return a, a.ctypes.data if a.size else None, a.size

    def reset(self, ids=None):
        """Restart the given streams (all when ids is None) from zero bytes."""
        self._check(self.n_streams)
        a, ptr, n = self._ids(ids)
        if a is not None and n == 0:
            return
        rc = _lib.acg_streams_reset(self._h, ptr, n)
        if rc:
            self._ac._raise(rc)

    def positions(self):
        """The bytes every stream has received: uint64 [n_streams]."""
        self._check(self.n_streams)
        pos = np.empty(self.n_streams, dtype=np.uint64)
        rc = _lib.acg_streams_positions(self._h, pos.ctypes.data)
        if rc:
            self._ac._raise(rc)
        return pos

    def _look(self, cands, ids):
        if not self._h:
            raise ValueError("the stream set is closed")
        if not isinstance(cands, Candidates) or not cands._h or cands._ac is not self._ac:
            raise ValueError("lookahead takes an open Candidates of this set's automaton")
        a, ptr, n = self._ids(ids)
        return a, ptr, n, (self.n_streams if a is None else n)

    def lookahead_np(self, cands, ids=None):
        """For every row -- stream ids[k], or every stream when ids is None -- and every candidate c of `cands`
        (AhoCorasick.candidates): whether feeding that stream c would return a match, as a bool array
        [rows, len(cands)].  No stream changes."""
        a, ptr, n, rows = self._look(cands, ids)
        out = np.empty((rows, cands.n), dtype=np.bool_)
        if rows == 0:  # an empty id list: no call, whose NULL ids would mean every stream
            return out
        rc = _lib.acg_streams_lookahead(self._h, cands._h, ptr, n, out.ctypes.data if out.size else None)
        if rc:
            self._ac._raise(rc)
        return out

    def lookahead_torch(self, cands, ids=None, device=None):
        """lookahead_np as a CUDA torch.bool tensor on the automaton's device (`device`, by default the current
        CUDA device).  Torch's current stream is synchronised first, as feed_torch does."""
        import torch
        a, ptr, n, rows = self._look(cands, ids)
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        out = torch.empty((rows, cands.n), dtype=torch.bool, device=dev)
        if rows == 0:
            return out
        torch.cuda.current_stream(dev).synchronize()
        rc = _lib.acg_streams_lookahead_devout(self._h, cands._h, ptr, n, out.data_ptr() if out.numel() else None)
        if rc:
            self._ac._raise(rc)
        return out


class Candidates:
    """A candidate set (include/acb200.h, acg_candidates_create): a fixed list of byte strings -- a tokenizer's
    vocabulary, say -- copied once to the automaton's device and reused by every lookahead of that automaton's
    stream sets.  Create it with AhoCorasick.candidates(); use it as a context manager or close() it."""

    def __init__(self, ac, cands):
        self._ac = ac
        self._h = None
        keep, ptr, _, on_dev, offs = _batch_input(cands)
        if on_dev:
            raise TypeError("candidates are given in host memory")
        h = _vp()
        rc = _lib.acg_candidates_create(ac._h, ptr if offs[-1] > offs[0] else None, offs.ctypes.data,
                                        offs.size - 1, C.byref(h))
        if rc:
            ac._raise(rc)
        self._h = h
        self.n = int(offs.size - 1)

    def __len__(self):
        return self.n

    def close(self):
        if self._h and _lib is not None:
            _lib.acg_candidates_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class Streams(_StreamSet):
    """A stream set (include/acb200.h, acg_streams_*): n_streams streams over one automaton, in find_iter mode
    (try_find_iter, Standard semantics) or overlapping mode (try_find_overlapping_iter).  A feed takes one chunk per
    stream -- in any form the batch calls take -- and returns, per stream, the matches of the mode's iterator over
    everything the stream has received whose end lies in this feed's bytes, offsets absolute within the stream.  A
    stream's matches over all its feeds, concatenated, are the iterator over its concatenated chunks.  One call at a
    time per set.  Create it with AhoCorasick.streams(); the automaton is kept alive by the set."""

    def __init__(self, ac, n_streams, overlapping=False):
        self._ac = ac
        self._h = None
        h = _vp()
        rc = _lib.acg_streams_create(ac._h, int(n_streams), int(bool(overlapping)), C.byref(h))
        if rc:
            ac._raise(rc)
        self._h = h
        self.n_streams = int(n_streams)
        self.overlapping = bool(overlapping)

    def feed_np(self, chunks):
        """One chunk per stream (a list of bytes / str, or (values, offsets) as the batch calls take): the new
        matches as a DOC_MATCH_DTYPE array, doc = the stream, ascending stream."""
        keep, ptr, n, on_dev, offs = _batch_input(chunks)
        self._check(offs.size - 1)
        cnt = _u64()
        return _until_it_fits(
            self._ac, max(self._ac._cap_hint, 64), lambda cap: np.empty(cap, DOC_MATCH_DTYPE), cnt,
            lambda out, cap: _lib.acg_streams_feed(self._h, ptr, on_dev, n, offs.ctypes.data, self.n_streams,
                                                   out.ctypes.data, cap, C.byref(cnt)))

    def feed(self, chunks):
        """One chunk per stream: one list of Match per stream."""
        return AhoCorasick._per_doc(self.feed_np(chunks), self.n_streams)

    def feed_torch(self, chunks):
        """(values, offsets) chunks with values a CUDA torch.uint8 tensor and offsets an int64 CUDA tensor on its
        device or a host array: the new matches as a BatchMatches of CUDA tensors, indexed by stream."""
        import torch
        values, keep, optr, n_chunks, on_dev = _torch_batch(chunks)
        self._check(n_chunks)
        match_offsets = torch.empty(n_chunks + 1, dtype=torch.int64, device=values.device)
        cnt = _u64()
        r = _until_it_fits(
            self._ac, self._ac._cap_hint, lambda cap: torch.empty((cap, 3), dtype=torch.int64, device=values.device),
            cnt, lambda records, cap: _lib.acg_streams_feed_devout(
                self._h, values.data_ptr(), values.numel(), optr, on_dev, self.n_streams, records.data_ptr(), cap,
                match_offsets.data_ptr(), C.byref(cnt)))
        return BatchMatches(r, match_offsets, r[:, 0] & 0xFFFFFFFF, r[:, 0] >> 32, r[:, 1], r[:, 2])


class ReplaceStreams(_StreamSet):
    """A replace set (include/acb200.h, acg_streams_create_replace): n_streams streams over one automaton (Standard
    semantics) whose text comes back with every find_iter match replaced by its pattern's replacement.  A feed takes
    one chunk per stream -- in any form Streams.feed* takes -- and returns per stream the bytes between the last
    feed's emit boundary and this one's: everything before the boundary is settled, the at most
    max_pattern_len - 1 bytes after it (held()) may still become part of a match.  flush() returns the held bytes
    of the given streams and restarts them.  A stream's outputs over its feeds, followed by its flush, are
    replace_all_bytes of its bytes.  The output is bytes: a boundary may fall inside a multi-byte UTF-8 character.
    One call at a time per set.  Create it with AhoCorasick.replace_streams()."""

    def __init__(self, ac, n_streams, replace_with):
        self._ac = ac
        self._h = None
        rkeep, rptr, roffs = ac._replacement_table(replace_with)
        h = _vp()
        rc = _lib.acg_streams_create_replace(ac._h, int(n_streams), rptr, roffs.ctypes.data, roffs.size - 1,
                                             C.byref(h))
        if rc:
            ac._raise(rc)
        self._h = h
        self.n_streams = int(n_streams)

    def feed_np(self, chunks):
        """One chunk per stream (a list of bytes / str, or (values, offsets) as the batch calls take): the released
        text as (values uint8, offsets uint64 [n_streams + 1]), stream s's at values[offsets[s]:offsets[s + 1]]."""
        keep, ptr, n, on_dev, offs = _batch_input(chunks)
        self._check(offs.size - 1)
        out_offsets = np.empty(self.n_streams + 1, dtype=np.uint64)
        values = self._ac._replace_until_it_fits(
            int(offs[-1]) - int(offs[0]), lambda cap: np.empty(cap, dtype=np.uint8),
            lambda out, cap, cnt: _lib.acg_streams_replace_feed(
                self._h, ptr, on_dev, n, offs.ctypes.data, self.n_streams, out.ctypes.data, cap,
                out_offsets.ctypes.data, cnt))
        return values, out_offsets

    def feed(self, chunks):
        """One chunk per stream: one bytes object per stream."""
        return self._split(*self.feed_np(chunks))

    def feed_torch(self, chunks):
        """(values, offsets) chunks with values a CUDA torch.uint8 tensor and offsets an int64 CUDA tensor on its
        device or a host array: the released text as (values, CUDA uint8; offsets, CUDA int64 [n_streams + 1])."""
        import torch
        values, keep, optr, n_chunks, on_dev = _torch_batch(chunks)
        self._check(n_chunks)
        dev = values.device
        span = values.numel() if on_dev else int(keep[-1]) - int(keep[0])
        out_offsets = torch.empty(n_chunks + 1, dtype=torch.int64, device=dev)
        out = self._ac._replace_until_it_fits(
            span, lambda cap: torch.empty(cap, dtype=torch.uint8, device=dev),
            lambda out, cap, cnt: _lib.acg_streams_replace_feed_devout(
                self._h, values.data_ptr(), values.numel(), optr, on_dev, self.n_streams, out.data_ptr(), cap,
                out_offsets.data_ptr(), cnt))
        return out, out_offsets

    def flush_np(self, ids=None):
        """The held bytes of the given streams (all when ids is None), raw, as (values uint8, offsets uint64
        [len(ids) + 1]); those streams then restart from zero bytes."""
        self._check(self.n_streams)
        a, ptr, k = self._ids(ids)
        if a is not None and k == 0:
            return np.empty(0, dtype=np.uint8), np.zeros(1, dtype=np.uint64)
        out_offsets = np.empty((self.n_streams if a is None else k) + 1, dtype=np.uint64)
        cnt = _u64()
        rc = _lib.acg_streams_flush(self._h, ptr, k, None, 0, out_offsets.ctypes.data, C.byref(cnt))
        while rc == E_OVERFLOW:  # the size query said how much; no stream was reset
            out = np.empty(int(cnt.value), dtype=np.uint8)
            rc = _lib.acg_streams_flush(self._h, ptr, k, out.ctypes.data, out.size, out_offsets.ctypes.data,
                                        C.byref(cnt))
            if rc == 0:
                return out, out_offsets
        if rc:
            self._ac._raise(rc)
        return np.empty(0, dtype=np.uint8), out_offsets

    def flush(self, ids=None):
        """The held bytes of the given streams (all when ids is None), one bytes object each; those streams then
        restart from zero bytes."""
        return self._split(*self.flush_np(ids))

    def held(self):
        """The bytes every stream holds back, uint64 [n_streams]: positions() - held() is its emit boundary."""
        self._check(self.n_streams)
        h = np.empty(self.n_streams, dtype=np.uint64)
        rc = _lib.acg_streams_held(self._h, h.ctypes.data)
        if rc:
            self._ac._raise(rc)
        return h

    @staticmethod
    def _split(values, offsets):
        b, o = values.tobytes(), offsets.tolist()
        return [b[o[i]:o[i + 1]] for i in range(len(o) - 1)]
