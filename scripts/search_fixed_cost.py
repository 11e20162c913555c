#!/usr/bin/env python
"""The fixed cost of the headline search: the part of each search's wall time that lies outside its games' simulation chains.

Builds the headline engine as bench.py does (CartPole, 4096 games, N = 50, synthetic weights seed 0, four rotating device
input batches, a 256 MiB L2 flush before every search) and reports, in one run:

  host split   scripts/search_host_split.py's parts of the wall time (prelude, enqueue, sync wait, device, epilogue, the
               trailing synchronise), and its torch.profiler pass: CUPTI kernel span against device_ms
  device split from a copy of the library built with -DMZ_FC_PHASES (scripts/fc_phase_split.py's build), the
               %globaltimer at which each CTA entered the kernel and each game started and finished, for one search:
                 start-up   first CTA entry -> first game start (tables and weights staged, first observation)
                 chain      first game start -> median game end
                 tail       median game end -> last game end
               (the instrumented kernel runs longer than the product one: set these against each other, and the
               product kernel's CUPTI span against device_ms)
  the tail     per warp (its two lock-stepped games) max(pair) - mean(pair) of the game durations (zero when the
               pair starts and ends together); per SM the games it
               held and its latest end; per game the tree levels and selection rounds per simulation, and how well they
               predict its duration

    python scripts/search_fixed_cost.py [--seconds 1.0] [--repeats 3] [--json OUT]

Needs a GPU; reads the card's name, power limit and SM clock in the same run and prints them with the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import fc_phase_split  # noqa: E402
import search_host_split  # noqa: E402

COLS = 11          # fc_search.cu's phase row: root..backup cycles, levels, rounds, sims, start ns, end ns, SM


def device_split(searches=3):
    """One instrumented search's per-game rows and per-CTA entry times (run in a child process: the library it loads is
    the instrumented copy)."""
    import torch
    from muzero_general_b200 import _lib
    _lib.LIB_PATH = fc_phase_split.build_instrumented(tempfile.mkdtemp(prefix="mz_fixed_cost_"))
    eng, search, flush = search_host_split.headline_engine()
    lib = eng.lib
    lib.mz_fc_phase_counters.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    lib.mz_fc_phase_rows.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
    lib.mz_fc_phase_ctas.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    B = eng.max_games
    for i in range(20):
        search(i)
    runs = []
    for i in range(searches):
        assert lib.mz_fc_phase_counters(None, 1) == 0
        flush.fill_(i & 0xFF)
        torch.cuda.synchronize()
        search(i)
        launch = eng.last_fc_launch
        rows = numpy.zeros((B, COLS), numpy.uint64)
        ctas = numpy.zeros(launch["grid"], numpy.uint64)
        ptr = lambda a: a.ctypes.data_as(C.POINTER(C.c_ulonglong))
        assert lib.mz_fc_phase_rows(ptr(rows), B, COLS) == 0
        assert lib.mz_fc_phase_ctas(ptr(ctas), launch["grid"]) == 0
        runs.append(analyse(rows.astype(numpy.int64), ctas.astype(numpy.int64), launch))
    eng.close()
    return runs


def analyse(rows, ctas, launch):
    us = lambda v: round(float(v) / 1000.0, 2)
    start, end, sm = rows[:, 8], rows[:, 9], rows[:, 10]
    dur = end - start
    entry = int(ctas.min())
    med_end = numpy.median(end)
    # lock-stepped pairs: the groups of a warp hold consecutive games (warp_first in fc_search.cu)
    pairs_per_warp = 32 // launch["group"]
    d = dur[: len(dur) // pairs_per_warp * pairs_per_warp].reshape(-1, pairs_per_warp)
    pair_excess = d.max(axis=1) - d.mean(axis=1)
    sms = numpy.unique(sm)
    games_per_sm = numpy.array([(sm == s).sum() for s in sms])
    last_per_sm = numpy.array([end[sm == s].max() for s in sms])
    sims = numpy.maximum(rows[:, 7], 1)
    levels, rounds = rows[:, 5] / sims, rows[:, 6] / sims
    slowest = int(numpy.argmax(end))
    return {
        "launch": launch,
        "startup_us": us(start.min() - entry),
        "cta_entry_spread_us": us(ctas.max() - entry),
        "chain_us": us(med_end - start.min()),
        "tail_us": us(end.max() - med_end),
        "first_entry_to_last_end_us": us(end.max() - entry),
        "duration_us": {"min": us(dur.min()), "median": us(numpy.median(dur)), "max": us(dur.max())},
        "start_spread_us": us(start.max() - start.min()),
        "pair_excess_us": {"median": us(numpy.median(pair_excess)), "p99": us(numpy.percentile(pair_excess, 99)),
                           "max": us(pair_excess.max())},
        "sms": int(len(sms)),
        "games_per_sm": {int(k): int(v) for k, v in zip(*numpy.unique(games_per_sm, return_counts=True))},
        "sm_last_end_after_median_end_us": {"min": us(last_per_sm.min() - med_end),
                                            "median": us(numpy.median(last_per_sm) - med_end),
                                            "max": us(last_per_sm.max() - med_end)},
        "sm_last_end_by_games_us": {int(k): us(numpy.median(last_per_sm[games_per_sm == k]) - med_end)
                                    for k in numpy.unique(games_per_sm)},
        "levels_per_sim": {"min": round(float(levels.min()), 3), "median": round(float(numpy.median(levels)), 3),
                           "max": round(float(levels.max()), 3)},
        "rounds_per_sim": {"min": round(float(rounds.min()), 3), "median": round(float(numpy.median(rounds)), 3),
                           "max": round(float(rounds.max()), 3)},
        "corr_duration_levels": round(float(numpy.corrcoef(dur, levels)[0, 1]), 3),
        "corr_duration_rounds": round(float(numpy.corrcoef(dur, rounds)[0, 1]), 3),
        "slowest_game": {"game": slowest, "duration_us": us(dur[slowest]), "levels_per_sim": round(float(levels[slowest]), 3),
                         "rounds_per_sim": round(float(rounds[slowest]), 3), "sm": int(sm[slowest]),
                         "games_on_its_sm": int((sm == sm[slowest]).sum()),
                         "partner_duration_us": us(dur[slowest ^ 1])},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--device-split-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("search_fixed_cost.py needs a CUDA device")
    if args.device_split_only:
        print(json.dumps(device_split()))
        return
    res = {"card": fc_phase_split.card()}
    res["host"] = [search_host_split.split_run(args.seconds) for _ in range(args.repeats)]
    res["profile"] = search_host_split.profile_run()
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--device-split-only"], stdout=subprocess.PIPE,
                           text=True, check=True)
    res["device"] = json.loads(child.stdout.strip().splitlines()[-1])
    res["card_after"] = fc_phase_split.card()

    print("| part (us per search) | " + " | ".join(f"run {k + 1}: median (p10-p90)" for k in range(args.repeats)) + " |")
    print("|---|" + "---|" * args.repeats)
    for p in search_host_split.PARTS + ("wall",):
        print(f"| {p} | " + " | ".join(f"{r['median_us'][p]:.1f} ({r['p10_us'][p]:.1f}-{r['p90_us'][p]:.1f})"
                                      for r in res["host"]) + " |")
    print("profile:", json.dumps(res["profile"]))
    for r in res["device"]:
        print(json.dumps(r))
    print("card:", res["card"], "after:", res["card_after"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
