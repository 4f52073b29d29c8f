"""Which engine every search call takes, on the dry-run build of the kernels (tests/emu/): the return code
and last_stats()["engine"] of each call under every engine override, on automata with and without a
prefilter plan, with anchored and unanchored input, and with `earliest` on leftmost automata.

`expected` below is the rule as the calls apply it:
- the prefilter engine can serve an input when the automaton has a plan, the input is unanchored, and
  `earliest` is not asked of a leftmost automaton (acg_find / acg_find_batch: unless the automaton has the
  packed prefilter, which makes an unanchored leftmost try_find ignore `earliest`);
- otherwise a call takes its other engine: the walk for the single-haystack overlapping and sharded calls,
  the sequential engine for the rest; an override of that other engine is honoured as is;
- an ACG_ENGINE_PREFILTER override the input cannot use is ACG_E_INVALID_ARG, except for acg_find and the
  sharded call, which fall back to the other engine."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import aho_corasick_b200 as ab  # noqa: E402
from aho_corasick_b200 import sharded as S  # noqa: E402
from test_emulated_batch import emulated_library  # noqa: E402,F401
from test_prefilter_plan import plan_of  # noqa: E402

WALK, PF, SEQ = int(ab.Engine.Walk), int(ab.Engine.Prefilter), int(ab.Engine.Sequential)
INVALID_ARG = -22
OVERLAPPING = ("overlapping", "overlapping_dev", "overlapping_devout", "count_overlapping_dev", "sharded",
               "sharded_dev", "overlapping_batch")
PER_INPUT = ("find_iter", "find_iter_dev", "find_iter_batch", "is_match_batch")
FIND = ("find", "find_batch")

HAY = np.frombuffer(b"xabcdx bcd cdeabcde--abcd" * 8, dtype=np.uint8).copy()
OFFS = np.array([0, 7, 7, 60, HAY.size], dtype=np.uint64)


def expected(call, override, auto):
    """(rc, engine) of `call` under `override` on automaton `auto`, for the input (anchored, earliest)."""
    has_plan, leftmost, packed, anchored, earliest = auto
    if call in FIND and earliest and not anchored and leftmost and packed:
        earliest = False
    pf_ok = has_plan and not anchored and not (earliest and leftmost)
    other = WALK if call in ("overlapping", "overlapping_dev", "overlapping_devout", "count_overlapping_dev",
                             "sharded", "sharded_dev") else SEQ
    if override == other:
        return 0, other
    if override == PF and not pf_ok and call not in ("find", "sharded", "sharded_dev"):
        return INVALID_ARG, None
    return 0, PF if pf_ok else other


def run(ac, call, anchored, earliest):
    """The call's return code."""
    lib, h, p, n = ab._lib, ac._h, HAY.ctypes.data, HAY.size
    cnt, ms, fnv, found = ctypes.c_uint64(), ctypes.c_float(), ctypes.c_uint64(), ctypes.c_int()
    out = np.zeros(4096, ab.MATCH_DTYPE)
    o, cap = out.ctypes.data, out.size
    flags = np.zeros(OFFS.size - 1, np.uint8)
    offs, nd = OFFS.ctypes.data, OFFS.size - 1
    if call == "overlapping":
        return lib.acg_find_overlapping(h, p, n, 0, n, anchored, o, cap, ctypes.byref(cnt))
    if call == "overlapping_dev":
        return lib.acg_find_overlapping_dev(h, p, n, 0, n, o, cap, ctypes.byref(cnt), ctypes.byref(ms))
    if call == "overlapping_devout":
        return lib.acg_find_overlapping_devout(h, p, n, 0, n, 20, 0, o, cap, ctypes.byref(cnt), ctypes.byref(ms))
    if call == "count_overlapping_dev":
        return lib.acg_count_overlapping_dev(h, p, n, 0, n, ctypes.byref(cnt), ctypes.byref(fnv), ctypes.byref(ms))
    if call == "find_iter":
        return lib.acg_find_iter(h, p, n, 0, n, anchored, o, cap, ctypes.byref(cnt))
    if call == "find_iter_dev":
        return lib.acg_find_iter_dev(h, p, n, 0, n, o, cap, ctypes.byref(cnt), ctypes.byref(ms))
    if call == "find":
        return lib.acg_find(h, p, n, 0, n, anchored, earliest, o, ctypes.byref(found))
    if call == "find_iter_batch":
        return lib.acg_find_iter_batch(h, p, 0, n, offs, nd, anchored, o, cap, ctypes.byref(cnt))
    if call == "overlapping_batch":
        return lib.acg_find_overlapping_batch(h, p, 1, n, offs, nd, anchored, o, cap, ctypes.byref(cnt))
    if call == "is_match_batch":
        return lib.acg_is_match_batch(h, p, 0, n, offs, nd, anchored, flags.ctypes.data)
    if call == "find_batch":
        return lib.acg_find_batch(h, p, 1, n, offs, nd, anchored, earliest, o, flags.ctypes.data)
    comm = S.Comm(S.unique_id(), 0, 1)
    try:
        comm.find_overlapping(ac, p, n, 0, (0, n), on_device=call == "sharded_dev")
        return 0
    except ab.DeviceError as e:
        return e.code
    finally:
        comm.close()


def automaton(kind, prefilter, empty):
    pats = [b"abcd", b"bcd", b"cde", b"xa"] + ([b""] if empty else [])
    return ab.AhoCorasick.builder().match_kind(kind).prefilter(prefilter).start_kind(ab.StartKind.Both) \
        .kind(ab.AhoCorasickKind.DFA).build(pats)


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("prefilter", [True, False])
@pytest.mark.parametrize("empty", [False, True])
def test_engine_choice(kind, prefilter, empty):
    ac = automaton(kind, prefilter, empty)
    has_plan = bool(plan_of(ac).supported)
    assert has_plan == (not empty)    # prefilter(False) keeps the plan: it is derived from the tables
    packed = ac.prefilter_kind() == 4
    assert packed == (kind != 0 and prefilter and not empty)
    calls = (OVERLAPPING if kind == 0 else ()) + PER_INPUT + FIND
    checked = 0
    for override in ab.Engine:
        ac.set_engine(override)
        for call in calls:
            for anchored in ((0,) if call in OVERLAPPING or call.endswith("_dev") else (0, 1)):
                for earliest in ((0, 1) if call in FIND else (0,)):
                    want_rc, want_engine = expected(call, int(override), (has_plan, kind != 0, packed, anchored, earliest))
                    ctx = (call, override.name, "anchored" if anchored else "unanchored", "earliest" if earliest else "")
                    rc = run(ac, call, anchored, earliest)
                    assert rc == want_rc, ctx
                    if rc == 0:
                        assert ac.last_stats()["engine"] == want_engine, ctx
                    checked += 1
    assert checked >= 4 * len(calls)
