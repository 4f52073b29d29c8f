"""The dense table built on the device (acg_build_on_device) against the host builder's, and searched
by both engines.  The switchable kernel variants (include/acb200_debug.h: ACG_EXP_KEY24,
ACG_EXP_STATIC_TILES, ACG_EXP_GLOBAL_TILES) are rows of tests/test_gpu_kernel_matrix.py."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_parity import assert_np_equal, to_device

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(900)
@pytest.mark.parametrize("cfg,kind,ci", [("cfg2", 0, False), ("cfg3", 1, True), ("cfg4", 2, False), ("cfg5", 0, False)])
def test_dense_table_built_on_the_device(cfg, kind, ci):
    """acg_build_on_device (SURVEY section 8f.2): the table filled by dfa_fill_level_kernel is bit-identical
    to the host builder's, and both engines search it with the oracle's results."""
    import torch
    c = W.CONFIGS[cfg]
    n_pat = min(c["n_patterns"], 30000)   # cfg5 at 30 000 patterns: 100 MB table, seconds for the oracle
    pats = W.make_patterns(n_pat, c["pattern_seed"])

    def builder():
        return ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA)
    host = builder().host_only(True).build(pats)
    dev = builder().device_fill(True).build(pats)
    th, td = host.tables(), dev.tables()
    for k in th:
        if isinstance(th[k], np.ndarray):
            assert np.array_equal(th[k], td[k]), (cfg, k)
        else:
            assert th[k] == td[k], (cfg, k)
    n = 8 << 20
    t = torch.empty(n, dtype=torch.uint8)
    W.torch_fill_config(cfg if cfg != "cfg5" else "cfg2", t, pats, chunk=1 << 24)
    hay = t.numpy()
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    d = to_device(t)
    assert_np_equal(dev.find_iter_dev_np(d.data_ptr(), n)[0], o.find_iter_np(hay), cfg)
    if kind == 0:
        want = o.find_overlapping_iter_np(hay)
        assert_np_equal(dev.find_overlapping_iter_dev_np(d.data_ptr(), n)[0], want, cfg)
        dev.set_engine(ab.Engine.Walk)
        assert_np_equal(dev.find_overlapping_iter_dev_np(d.data_ptr(), n)[0], want, (cfg, "walk"))
