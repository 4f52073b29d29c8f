"""Dry-run shim for the `-m gpu` suite (test infrastructure, never used by the product).

With ACB_FAKE_DEVICE=1 the host-buffer search entry points of libacb200.so (acg_find_iter,
acg_find_overlapping, acg_find and their packed counterparts) are answered by the CPU oracle
instead of the CUDA kernels, on handles built with the real host-side builder.  That lets the GPU
test *programs* and the Python mirror (argument marshalling, Input handling, overflow protocol,
replace/stream glue, packed wrapper) be exercised on a machine without a GPU:

    ACB_FAKE_DEVICE=1 python -m pytest tests/test_gpu_zz_packed.py tests/test_gpu_parity.py -k "..."

Tests that use device-resident haystacks (torch.cuda, *_dev entry points) cannot run this way.
A pass here says nothing about the kernels; the real `-m gpu` run on an H100 does.
"""
import ctypes as C

import numpy as np

import aho_corasick_b200 as ab
import oracle_py as O

_registry = {}   # handle value -> dict(oracle=..., packed=bool)
E_OVERFLOW, E_INVALID_SPAN = -21, -20


def _patterns(arr, lens, n):
    addrs = C.cast(arr, C.POINTER(C.c_void_p))  # raw addresses: c_char_p indexing would stop at NUL bytes
    return [C.string_at(addrs[i], lens[i]) if lens[i] else b"" for i in range(n)]


def install():
    lib = ab._lib
    real_build_host = lib.acg_build_host
    real_packed_build_host = lib.acg_packed_build_host
    real_match_errors = {}

    def acg_build(arr, lens, n, opts_ref, out_ref):
        rc = real_build_host(arr, lens, n, opts_ref, out_ref)
        if rc == 0:
            o = opts_ref._obj
            pats = _patterns(arr, lens, n)
            _registry[out_ref._obj.value] = dict(
                oracle=O.Oracle(pats, match_kind=o.match_kind, start_kind=o.start_kind,
                                ascii_case_insensitive=bool(o.ascii_case_insensitive),
                                byte_classes=bool(o.byte_classes), prefilter=bool(o.prefilter), kind=O.KIND_DFA),
                match_kind=o.match_kind, start_kind=o.start_kind)
        return rc

    def acg_packed_build(arr, lens, n, cfg_ref, out_ref):
        rc = real_packed_build_host(arr, lens, n, cfg_ref, out_ref)
        if rc == 0 and out_ref._obj.value:
            c = cfg_ref._obj
            _registry[("packed", out_ref._obj.value)] = dict(
                oracle=O.Oracle(_patterns(arr, lens, n), match_kind=c.match_kind, kind=O.KIND_DFA),
                match_kind=c.match_kind, start_kind=0)
        return rc

    def _validate(ent, n, s, e, anchored, overlapping):
        # mirrors validate_common / overlapping_impl / find_iter_impl in csrc/acb_api.cu
        if not (e <= n and s <= e + 1):
            return E_INVALID_SPAN
        sk = ent["start_kind"]
        if sk == 0 and anchored:
            return -10
        if sk == 1 and not anchored:
            return -11
        if overlapping and ent["match_kind"] != 0:
            return -13
        return 0

    def _hay(ptr, n):
        return np.frombuffer(C.string_at(ptr, n) if n else b"", dtype=np.uint8)

    def _emit(r, out_addr, cap, cnt_ref):
        cnt_ref._obj.value = len(r)
        if len(r) > cap:
            return E_OVERFLOW
        if len(r):
            dst = np.ctypeslib.as_array(C.cast(out_addr, C.POINTER(C.c_uint8)), (cap * 24,)).view(ab.MATCH_DTYPE)
            dst["pid"][:len(r)] = r["pid"]
            dst["_pad"][:len(r)] = 0
            dst["start"][:len(r)] = r["start"]
            dst["end"][:len(r)] = r["end"]
        return 0

    def _iter(key, overlapping):
        def fn(h, ptr, n, s, e, anchored, out_addr, cap, cnt_ref):
            ent = _registry[key(h)]
            rc = _validate(ent, n, s, e, anchored, overlapping)
            cnt_ref._obj.value = 0
            if rc:
                return rc
            o = ent["oracle"]
            f = o.find_overlapping_iter_np if overlapping else o.find_iter_np
            return _emit(f(_hay(ptr, n), span=(s, e), anchored=bool(anchored)), out_addr, cap, cnt_ref)
        return fn

    def _hval(h):
        return h.value if hasattr(h, "value") else h

    def _find(key):
        def fn(h, ptr, n, s, e, anchored, earliest, out_addr, found_ref):
            ent = _registry[key(h)]
            found_ref._obj.value = 0
            rc = _validate(ent, n, s, e, anchored, False)
            if rc:
                return rc
            m = ent["oracle"].try_find(_hay(ptr, n), span=(s, e), anchored=bool(anchored), earliest=bool(earliest))
            if m is not None:
                dst = np.ctypeslib.as_array(C.cast(out_addr, C.POINTER(C.c_uint8)), (24,)).view(ab.MATCH_DTYPE)
                dst["pid"][0], dst["start"][0], dst["end"][0] = m
                found_ref._obj.value = 1
            return 0
        return fn

    lib.acg_build = acg_build
    lib.acg_find_iter = _iter(_hval, False)
    lib.acg_find_overlapping = _iter(_hval, True)
    lib.acg_find = _find(_hval)
    lib.acg_packed_build = acg_packed_build
    pk = lambda h: ("packed", _hval(h))  # noqa: E731
    it = _iter(pk, False)
    lib.acg_packed_find_iter = lambda h, ptr, n, s, e, out, cap, cnt: it(h, ptr, n, s, e, 0, out, cap, cnt)
    fd = _find(pk)
    lib.acg_packed_find = lambda h, ptr, n, s, e, out, found: fd(h, ptr, n, s, e, 0, 0, out, found)
