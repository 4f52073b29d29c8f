#!/usr/bin/env python3
"""How often each part of the stride-2 prefilter step runs on cfg 2 and cfg 3 (CPU only, no GPU).

    python tools/step_counts.py [--mib 64] [--workloads cfg2,cfg3]

Restates the first-stage probe of prefilter_kernel (as tests/test_prefilter_plan.py does) over the
first MiB of each workload's haystack and reports, per warp step of 1 KiB and of 2 KiB: first-stage
hits, second-stage rounds (32 items per round, two items per hit), trips of the per-lane slot loop
(the largest hit count of any lane) and steps that take the unselective path (more hits than the
slots hold, or a lane with more than 7).  Multiplied with the instruction counts of the SASS sections
(DESIGN.md section 3) this gives dynamic warp instructions per KiB -- a count, not a time.
For the 2 KiB step it also prints the distribution of hits per step (quantiles, the largest count,
steps over 48 and over 64 hits): what a smaller slot queue per warp would have to hold.
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

SLOTS = 256  # slot capacity per warp step (prefilter_kernel's kPfSlots)


def counts(wl, mib):
    import aho_corasick_b200 as ab
    from aho_corasick_b200 import workload as W
    from test_prefilter_plan import plan_of

    pats, hay, _ = W.make_config(wl, mib << 20)
    b = ab.AhoCorasick.builder().host_only().kind(ab.AhoCorasickKind.DFA)
    if wl == "cfg3":
        b.ascii_case_insensitive(True).match_kind(ab.MatchKind.LeftmostFirst)
    ac = b.build(pats)
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
    res = {"workload": wl, "mib": mib, "first_stage_pass_rate": float(hit.mean())}
    for step in (1024, 2048):
        n_steps = n // step
        hs = hit[: n_steps * step // 2].reshape(n_steps, step // 512, 32, 8)  # [step][group][lane][probe]
        per_lane = hs.sum(axis=(1, 3))                                      # [step][lane]
        hits = per_lane.sum(axis=1)
        res[f"step_{step}"] = {
            "steps": int(n_steps),
            "hits_per_step": float(hits.mean()),
            "steps_with_hits": float((hits > 0).mean()),
            "second_stage_rounds_per_step": float(np.ceil(2 * np.minimum(hits, SLOTS) / 32).mean()),
            "slot_loop_trips_per_step": float(per_lane.max(axis=1).mean()),
            "unselective_steps": float(((hits > SLOTS) | (per_lane.max(axis=1) > 7)).mean()),
        }
        if step == 2048:
            q = np.percentile(hits, [50, 90, 99, 99.9, 99.99])
            res[f"step_{step}"]["hits_distribution"] = {
                "p50": float(q[0]), "p90": float(q[1]), "p99": float(q[2]), "p99.9": float(q[3]), "p99.99": float(q[4]),
                "max": int(hits.max()), "steps_over_64": int((hits > 64).sum()),
                "steps_over_48": int((hits > 48).sum()), "lanes_over_7": int((per_lane.max(axis=1) > 7).sum()),
            }
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    ap.add_argument("--workloads", default="cfg2,cfg3")
    args = ap.parse_args()
    print(json.dumps([counts(wl, args.mib) for wl in args.workloads.split(",")], indent=1))


if __name__ == "__main__":
    main()
