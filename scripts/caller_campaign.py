#!/usr/bin/env python
"""GPU campaign: the batched callers around the scan (propose_gridpoints, BatchTOPPRA on common / per-path / proposed grids,
TOPPRAsd and sd_bisect, reachable and controllable sets, the output parametrizers, the constraint producers) against the
oracle-backed engine double on randomly shaped problems, for as long as wanted.  The checks are those of
tests/test_zzz_caller_campaign.py; every mismatching seed is printed, and at the end the problem count and the branch
histogram.

usage: python scripts/caller_campaign.py [--minutes M] [--seed S]          (needs a CUDA device and a built package)"""
import argparse
import os
import sys
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import pytest  # noqa: E402
import torch  # noqa: E402

import test_zzz_caller_campaign as cc  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=5.0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the caller campaign needs a CUDA device"
    patch = pytest.MonkeyPatch()
    ta = cc.Side(True, patch)
    t_end = time.time() + 60 * args.minutes
    seed, bad, hist = args.seed, [], {}
    t_report = time.time() + 60
    while time.time() < t_end:
        try:
            if seed % 50 == 49:
                cc.check_large(ta, seed, hist)
            cc.check_problem(ta, seed, hist, seed)
        except Exception as e:          # a mismatch, or a call that raised where it should not have
            bad.append(seed)
            print("MISMATCH seed %d: %s: %s" % (seed, type(e).__name__, (str(e).splitlines() or [""])[0][:300]),
                  flush=True)
            traceback.print_exc(limit=3)
        seed += 1
        if time.time() > t_report:      # a progress line a minute
            t_report += 60
            print("%d problems, %d mismatches" % (seed - args.seed, len(bad)), flush=True)
    patch.undo()
    print("problems: %d (seeds %d..%d), mismatches: %d %s" % (seed - args.seed, args.seed, seed - 1, len(bad), bad))
    print("branches: %s" % sorted(hist.items()))
    missing = [k for k in cc.FLOORS if not hist.get(k)]
    if missing:
        print("branches never reached: %s" % missing)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
