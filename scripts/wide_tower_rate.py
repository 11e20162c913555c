"""Gomoku's 6 x 128-channel towers on the wide x3 tensor-core route (MZ_TC_WIDE=1) next to the fp32 CUDA-core route, in one
process, with synthetic weights (seed 0; the rates do not depend on them):

  tower     kernel time of one tower at the in-search dynamics site (stem + 6 blocks = 13 convs, boards gathered from a
            pool) for 128 and 1024 boards on 11 x 11, with the algorithmic TFLOP/s (2 x 9 x 128 x cin per position and
            conv, counted once although the x3 recipe issues three MMAs).  The wide route is one conv_tower_wide_kernel
            launch (mz_debug_wide_tower); the CUDA-core route is its 13 conv3x3_kernel launches (one 129 -> 128 conv and
            twelve 128 -> 128 convs, timed through mz_debug_conv3x3).  Each is timed --reps times (CUDA events of
            mz_kernel_timing); median, min and max are printed.
  search    one 128-game N = 400 search: wall time (the mean of 2 after a warm-up, graph replay on) and the kernel split
            of one more search with mz_kernel_timing on.
  selfplay  SelfPlay.play_moves env-steps/s on the device loop, 128 games, N = 400, 1 warm-up move + 3 timed moves.

--side S (default 11) puts the net on S x S boards (games.gomoku.MuZeroConfig(board_size=S)).  --route pair measures the CTA-pair
kernel (conv_tower_wide_pair_kernel through mz_debug_wide_pair_tower; MZ_TC_WIDE=2 for the search and the device loop) in
place of the one-CTA kernel: at sides the one-CTA plan refuses (15, 16) against the CUDA cores as above, and at 11 x 11, for
information, its tower alone against the one-CTA kernel's, in two rounds that alternate the routes.

Prints one JSON line per measurement and a last line with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

from device_games_rate import card, rate  # noqa: E402

C, BLOCKS = 128, 6
H = W = 11


def tower_flops(n):
    return 2.0 * 9 * C * n * H * W * ((C + 1) + 2 * BLOCKS * C)


def _timed(eng, fn, reps, cls):
    """[ms] of the kernels of class `cls` per call of fn, reps calls after one warm-up."""
    fn()
    eng.kernel_times()
    out = []
    for _ in range(reps):
        fn()
        out.append(eng.kernel_times()[cls][0])
    return out


def towers(eng, reps, routes=("wide_x3", "cuda_core"), rounds=1):
    from muzero_general_b200.engine import debug_conv3x3, debug_wide_pair_tower, debug_wide_tower
    rs = numpy.random.RandomState(0)
    A = H * W
    for n in (128, 1024):
        x = rs.standard_normal((n, C, H, W)).astype(numpy.float32)
        ws = [(rs.standard_normal((C, C + 1 if i == 0 else C, 3, 3)) / 34).astype(numpy.float32) for i in range(1 + 2 * BLOCKS)]
        bs = [numpy.zeros(C, numpy.float32) for _ in ws]
        act = rs.randint(0, A, n).astype(numpy.int32)
        par = numpy.zeros(n, numpy.int32)
        xs = numpy.concatenate([x, numpy.zeros((n, 1, H, W), numpy.float32)], 1)

        def timed(route):
            if route == "cuda_core":
                stem = _timed(eng, lambda: debug_conv3x3(xs, ws[0], bs[0], relu=True), reps, "conv3x3_kernel")
                body = _timed(eng, lambda: debug_conv3x3(x, ws[1], bs[1], relu=True), reps, "conv3x3_kernel")
                return [s + 2 * BLOCKS * b for s, b in zip(stem, body)]
            fn = debug_wide_pair_tower if route == "pair_x3" else debug_wide_tower
            return _timed(eng, lambda: fn(x, ws, bs, site="dynamics_pool", actions=act, A=A, parents=par, pool_stride=1),
                          reps, "conv_tower_tc_kernel")

        for k in range(rounds):
            for route in routes:
                ms = timed(route)
                med = float(numpy.median(ms))
                print(json.dumps({"measure": "tower_dynamics_pool", "route": route, **({"side": H} if H != 11 else {}), "boards": n, "reps": reps,
                                  **({"round": k} if rounds > 1 else {}),
                                  "ms_median": round(med, 4), "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
                                  "tflops": round(tower_flops(n) / (med * 1e-3) / 1e12, 2)}), flush=True)


def search(cfg, weights, route):
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.netspec import netspec_from_config
    spec = netspec_from_config(cfg)
    obs = numpy.random.RandomState(1).randint(0, 2, size=(128, spec.obs_elems)).astype(numpy.float32)
    eng = SearchEngine(cfg, max_games=128, num_simulations=400)
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
    eng.kernel_timing(False)
    print(json.dumps({"measure": "search_128x400", "route": route, "numerics": eng.numerics, "wall_ms": round(wall, 1),
                      "kernel_ms_launches": split}), flush=True)
    eng.close()


def main():
    global H, W
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--skip-selfplay", action="store_true")
    ap.add_argument("--side", type=int, default=11, help="board side of the Gomoku net (11, 15 or 16)")
    ap.add_argument("--route", choices=("wide", "pair"), default="wide",
                    help="tensor-core route: the one-CTA kernel (MZ_TC_WIDE=1) or CTA pairs (MZ_TC_WIDE=2)")
    args = ap.parse_args()
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    H = W = args.side
    name, power = card()
    mod = load_game_module("gomoku")
    cfg = mod.MuZeroConfig(board_size=args.side)
    weights = synthetic_weights(netspec_from_config(cfg), 0)
    tc_route, switch = ("pair_x3", "2") if args.route == "pair" else ("wide_x3", "1")
    probe = SearchEngine(cfg, max_games=1, num_simulations=1)       # a handle to switch mz_kernel_timing on
    probe.kernel_timing(True)
    if args.route == "pair" and args.side == 11:                    # for information: the pair against one CTA
        towers(probe, args.reps, ("pair_x3", "wide_x3"), rounds=2)
    else:
        towers(probe, args.reps, (tc_route, "cuda_core"))
    probe.kernel_timing(False)
    probe.close()
    for route in (tc_route, "cuda_core"):
        if args.route == "pair" and args.side == 11:
            break
        if route == tc_route:
            os.environ["MZ_TC_WIDE"] = switch
        else:
            os.environ.pop("MZ_TC_WIDE", None)
        search(cfg, weights, route)
        if not args.skip_selfplay:
            c = mod.MuZeroConfig(board_size=args.side)
            c.rng_mode, c.num_parallel_games = "philox", 128
            r, steps, dt = rate(mod, c, weights, True, 1, 3, 0.0)
            print(json.dumps({"measure": "selfplay_device_128x400", "route": route, "env_steps_per_s": round(r, 2),
                              "env_steps": steps, "seconds": round(dt, 2)}), flush=True)
    os.environ.pop("MZ_TC_WIDE", None)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
