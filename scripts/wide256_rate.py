"""games/atari.py's 16 x 256-channel towers on the 256-channel x3 tensor-core route (MZ_TC_WIDE=3) next to the fp32 CUDA-core
route, in one process, with synthetic weights (seed 0; the rates do not depend on them):

  tower     kernel time of the 33-conv dynamics tower at the in-search site (stem + 16 blocks on the 6 x 6 hidden board,
            boards gathered from a pool) for 128 and 1024 boards, with the algorithmic TFLOP/s (2 x 9 x 256 x cin per
            position and conv, counted once although the x3 recipe issues three MMAs).  The tensor-core route is one
            conv_tower_wide256_kernel launch (mz_debug_wide256_tower); the CUDA-core route is its 33 conv3x3_kernel launches
            (one 257 -> 256 conv and 32 256 -> 256 convs, timed through mz_debug_conv3x3).  Each is timed --reps times
            (CUDA events of mz_kernel_timing); median, min and max are printed.  For the tensor-core route also the L2
            weight traffic the plan implies: each CTA of a pair streams its 128-output-channel half of every layer's x3
            image (36 stages x 32 KB), once per group of `boards` boards.
  search    one N = 50 search of --games games (128, and 1024 with --games 128,1024): wall time (the mean of 2 after a
            warm-up, graph replay on) and the mz_kernel_timing split of one more search by kernel class (tree, tower,
            heads, conv, other, ...).  On the tensor-core route `conv` is the DownSample stem alone; on the CUDA-core route
            it also holds the tower convs, so the stem's share is printed from a separately timed initial_inference on
            the tensor-core route (the stem's kernels are the same on both routes).

Prints one JSON line per measurement and a last line with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

from device_games_rate import card  # noqa: E402
from wide_tower_rate import _timed  # noqa: E402

C, BLOCKS, H, W = 256, 16, 6, 6
LAYERS = 1 + 2 * BLOCKS
STAGE_BYTES, STAGES = 32768, 36


def tower_flops(n):
    return 2.0 * 9 * C * n * H * W * ((C + 1) + 2 * BLOCKS * C)


def towers(eng, reps, sizes=(128, 1024)):
    from muzero_general_b200.engine import debug_conv3x3, debug_wide256_tower, debug_wide256_tower_plan
    rs = numpy.random.RandomState(0)
    A = 18
    for n in sizes:
        x = rs.standard_normal((n, C, H, W)).astype(numpy.float32)
        ws = [(rs.standard_normal((C, C + 1 if i == 0 else C, 3, 3)) / 48).astype(numpy.float32) for i in range(LAYERS)]
        bs = [numpy.zeros(C, numpy.float32) for _ in ws]
        act = rs.randint(0, A, n).astype(numpy.int32)
        par = numpy.zeros(n, numpy.int32)
        xs = numpy.concatenate([x, numpy.zeros((n, 1, H, W), numpy.float32)], 1)
        plan, why = debug_wide256_tower_plan(n, C, H, W, BLOCKS, True, eng_sms())
        assert plan, why
        for route in ("wide256_x3", "cuda_core"):
            if route == "cuda_core":
                stem = _timed(eng, lambda: debug_conv3x3(xs, ws[0], bs[0], relu=True), reps, "conv3x3_kernel")
                body = _timed(eng, lambda: debug_conv3x3(x, ws[1], bs[1], relu=True), reps, "conv3x3_kernel")
                ms = [s + 2 * BLOCKS * b for s, b in zip(stem, body)]
            else:
                ms = _timed(eng, lambda: debug_wide256_tower(x, ws, bs, site="dynamics_pool", actions=act, A=A, parents=par,
                                                             pool_stride=1), reps, "conv_tower_tc_kernel")
            med = float(numpy.median(ms))
            rec = {"measure": "tower_dynamics_pool", "route": route, "boards": n, "reps": reps, "ms_median": round(med, 4),
                   "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
                   "tflops": round(tower_flops(n) / (med * 1e-3) / 1e12, 2)}
            if route == "wide256_x3":
                groups = -(-n // plan["boards"])
                weight_bytes = LAYERS * 2 * STAGES * STAGE_BYTES * groups
                rec.update(boards_per_pair=plan["boards"], l2_weight_TBps=round(weight_bytes / (med * 1e-3) / 1e12, 2))
            print(json.dumps(rec), flush=True)


def eng_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def search(cfg, weights, route, games):
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.netspec import netspec_from_config
    spec = netspec_from_config(cfg)
    obs = numpy.random.RandomState(1).random_sample((games, spec.obs_elems)).astype(numpy.float32)
    eng = SearchEngine(cfg, max_games=games, num_simulations=50)
    eng.load_weights(weights)
    eng.search(obs=obs, add_exploration_noise=False)
    t0 = time.perf_counter()
    for _ in range(2):
        eng.search(obs=obs, add_exploration_noise=False)
    wall = (time.perf_counter() - t0) / 2 * 1e3
    eng.kernel_timing(True)
    eng.kernel_times()
    eng.search(obs=obs, add_exploration_noise=False)
    split = {k: [round(ms, 2), cnt] for k, (ms, cnt) in eng.kernel_times().items() if cnt}
    rec = {"measure": f"search_{games}x50", "route": route, "numerics": eng.numerics, "wall_ms": round(wall, 1),
           "kernel_ms_launches": split}
    if route == "wide256_x3":                         # the DownSample stem alone: the conv class of initial_inference
        eng.initial_inference(obs)
        eng.kernel_times()
        eng.initial_inference(obs)
        rec["stem_conv_ms"] = round(eng.kernel_times()["conv3x3_kernel"][0], 2)
    eng.kernel_timing(False)
    print(json.dumps(rec), flush=True)
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--games", default="128", help="comma-separated search batch sizes, e.g. 128,1024")
    ap.add_argument("--skip-search", action="store_true")
    args = ap.parse_args()
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    cfg = load_game_module("atari").MuZeroConfig()
    weights = synthetic_weights(netspec_from_config(cfg), 0)
    probe = SearchEngine(load_game_module("gomoku").MuZeroConfig(), max_games=1, num_simulations=1)   # mz_kernel_timing switch
    probe.kernel_timing(True)
    towers(probe, args.reps)
    probe.kernel_timing(False)
    probe.close()
    if not args.skip_search:
        for games in (int(g) for g in args.games.split(",")):
            for route in ("wide256_x3", "cuda_core"):
                if route == "wide256_x3":
                    os.environ["MZ_TC_WIDE"] = "3"
                else:
                    os.environ.pop("MZ_TC_WIDE", None)
                search(cfg, weights, route, games)
    os.environ.pop("MZ_TC_WIDE", None)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
