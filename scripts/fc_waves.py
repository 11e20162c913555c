#!/usr/bin/env python
"""Kernel time of the headline fused FC search (CartPole, N = 50, synthetic weights seed 0, inputs seeded like bench.py's)
at batch sizes on either side of what one wave of resident CTAs holds.

A persistent grid runs every game whose slot is resident in the first wave; the rest wait for a slot to free up and
run a second chain of N dependent simulations after it.  On 132 SMs, 64-thread CTAs hold 3696 of these games and
128- or 256-thread CTAs 4224, so with MZ_FC_THREADS=64 a second pass shows up as a step in time between 3169 and 4096
games, and with the planned CTA size it does not.

    python scripts/fc_waves.py [--games 3168 3169 4096 4224] [--searches 20] [--json OUT]

Prints one line per batch size (median, minimum and maximum device time of the search, the launch's grid, block and
CTAs per SM) and the card and power limit it ran on.  Needs a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fc_phase_split import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, nargs="+", default=[3168, 3169, 4096, 4224])
    ap.add_argument("--searches", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    N, B = 50, max(args.games)
    cfg = load_game_module("cartpole").MuZeroConfig()
    spec = netspec_from_config(cfg)
    rs = numpy.random.RandomState(100)
    obs = rs.uniform(-0.05, 0.05, size=(B, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * spec.action_space, size=B)
    game_id = numpy.arange(B, dtype=numpy.int64)

    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=cfg.seed)
    eng.load_weights(synthetic_weights(spec, 0))
    results = {"card": card(), "num_simulations": N, "points": []}
    for n in args.games:
        run = lambda: eng.search(obs=obs[:n], add_exploration_noise=True, noise=noise[:n], game_id=game_id[:n])
        for _ in range(3):
            run()
        ms = sorted(run().device_ms for _ in range(args.searches))
        p = {"games": n, "kernel_ms": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1]}
        if hasattr(eng, "last_fc_launch"):                       # absent from builds before the residency planner
            p.update(eng.last_fc_launch or {})
        results["points"].append(p)
        launch = (f"  grid {p['grid']} x {p['block']} threads, {p['ctas_per_sm']} CTAs/SM, {p['smem']} B shared"
                  if "grid" in p else "")
        print(f"{n:6d} games: {p['kernel_ms']:.4f} ms (min {p['min_ms']:.4f}, max {p['max_ms']:.4f}, "
              f"{args.searches} searches){launch}")
    eng.close()
    print("card:", results["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
