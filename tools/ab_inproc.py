#!/usr/bin/env python3
"""In-process A/B of kernel variants (one haystack fill, many `acg_debug_set_experiment` settings).

    python tools/ab_inproc.py --workload cfg2 --exps 0,1,16,17 [--hay-gib 4] [--steps 8] [--engine 0]

Prints one JSON line per variant: best / mean scan_ms of the scan kernel (CUDA events inside the
library), the match count and the FNV of the ordered stream (must agree across variants).
"""
import argparse
import ctypes
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--exps", default="0")
    ap.add_argument("--hay-gib", type=float, default=4.0)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--engine", type=int, default=0)
    ap.add_argument("--device-fill", action="store_true")
    args = ap.parse_args()
    import time
    import torch
    import aho_corasick_b200 as ab
    from aho_corasick_b200 import workload as W

    cfg = W.CONFIGS[args.workload]
    pats = W.config_patterns(args.workload)
    b = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA)
    if args.workload == "cfg3":
        b.ascii_case_insensitive(True).match_kind(ab.MatchKind.LeftmostFirst)
    if args.workload == "cfg4":
        b.match_kind(ab.MatchKind.LeftmostFirst)
    if args.device_fill:
        b.device_fill(True)
    t0 = time.perf_counter()
    ac = b.build(pats).set_engine(args.engine)
    build_s = time.perf_counter() - t0
    n = int(args.hay_gib * (1 << 30))
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config(args.workload, d_hay, pats)
    torch.cuda.synchronize()
    overlapping = args.workload in ("cfg2", "cfg5", "cfg2b")
    ab._lib.acg_debug_set_experiment.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
    for exp in [int(x) for x in args.exps.split(",")]:
        assert ab._lib.acg_debug_set_experiment(ac._h, exp) == 0
        ms_list, res = [], None
        try:
            for i in range(args.steps + 2):
                if overlapping:
                    cnt, fnv, _ = ac.count_overlapping_dev(d_hay.data_ptr(), n)
                    res = (cnt, fnv)
                else:
                    r, _ = ac.find_iter_dev_np(d_hay.data_ptr(), n)
                    res = (len(r), int(r["end"].astype("uint64").sum() ^ r["pid"].astype("uint64").sum()))
                st = ac.last_stats()
                if i >= 2:
                    ms_list.append(st["scan_ms"])
            print(json.dumps({"workload": args.workload, "exp": exp, "engine": int(st["engine"]),
                              "scan_ms_best": min(ms_list), "scan_ms_mean": sum(ms_list) / len(ms_list),
                              "order_ms": st["order_ms"], "candidates": int(st["candidates"]),
                              "matches": res[0], "check": res[1], "gib": args.hay_gib, "build_s": build_s,
                              "gbs_best": n / (min(ms_list) * 1e-3) / 1e9}), flush=True)
        except Exception as e:  # keep going: one broken variant must not cost the trip
            print(json.dumps({"workload": args.workload, "exp": exp, "error": repr(e)}), flush=True)


if __name__ == "__main__":
    main()
