#!/usr/bin/env python3
"""How often each part of the stride-2 prefilter step runs on cfg 2 (CPU only, no GPU).

    python tools/step_counts.py [--mib 64]

Restates the first-stage probe of prefilter_kernel (as tests/test_prefilter_plan.py does) over the
first MiB of the cfg 2 haystack and reports, per warp step of 1 KiB and of 2 KiB: first-stage hits,
second-stage rounds (32 items per round, two items per hit), trips of the per-lane slot loop (the
largest hit count of any lane) and steps that overflow the 256 slots.  Multiplied with the
instruction counts of the SASS sections (DESIGN.md section 3) this gives dynamic warp instructions
per KiB -- a count, not a time.
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    args = ap.parse_args()
    import aho_corasick_b200 as ab
    from aho_corasick_b200 import workload as W
    from test_prefilter_plan import plan_of

    pats, hay, _ = W.make_config("cfg2", args.mib << 20)
    ac = ab.AhoCorasick.builder().host_only().kind(ab.AhoCorasickKind.DFA).build(pats)
    p = plan_of(ac)
    assert p.stride == 2 and not p.dense and not p.wide
    bitmap = np.ctypeslib.as_array(C.cast(p.bitmap, C.POINTER(C.c_uint32)), shape=(int(p.bitmap_words),)).copy()
    h = hay[: (hay.size // 2048) * 2048].astype(np.uint32)
    n = h.size - 4
    pos = np.arange(0, n, 2)  # even offsets: the stride-2 first stage
    win = h[pos] | (h[pos + 1] << 8) | (h[pos + 2] << 16) | (h[pos + 3] << 24)
    gm = (win | (p.fold & 0x00FFFFFF)) & 0xFFFFFFFF
    mult8 = (p.mult3 << p.key_shift) & 0xFFFFFFFF
    hh = (gm.astype(np.uint64) * mult8) & 0xFFFFFFFF
    bit = (hh >> p.shift) * 8 + (gm & 7)
    hit = ((bitmap[(bit >> 5).astype(np.int64)] >> (bit & 31).astype(np.uint32)) & 1).astype(np.int64)
    # lane L of a step owns the 16-byte groups at g * 512 + 16 L: 8 probes per group
    res = {"mib": args.mib, "first_stage_pass_rate": float(hit.mean())}
    for step in (1024, 2048):
        n_steps = n // step
        hs = hit[: n_steps * step // 2].reshape(n_steps, step // 512, 32, 8)  # [step][group][lane][probe]
        per_lane = hs.sum(axis=(1, 3))                                      # [step][lane]
        hits = per_lane.sum(axis=1)
        res[f"step_{step}"] = {
            "hits_per_step": float(hits.mean()),
            "steps_with_hits": float((hits > 0).mean()),
            "second_stage_rounds_per_step": float(np.ceil(2 * np.minimum(hits, 256) / 32).mean()),
            "slot_loop_trips_per_step": float(per_lane.max(axis=1).mean()),
            "unselective_steps": float(((hits > 256) | (per_lane.max(axis=1) > 7)).mean()),
        }
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
