"""Gomoku on 11 x 11 (121 actions, four children per lane in the tree step) next to 15 x 15 (225 actions, eight per
lane): env-steps/s of SelfPlay.play_moves on the device loop and on the host loop at the same batch, in one process, and
the per-kernel-class device times of one search at each size (mz_kernel_times), so the tree step's share shows.

    python scripts/wide_actions_rate.py                      # the shipped 6 x 128-channel towers, N = 400, 128 games
    python scripts/wide_actions_rate.py --sims 50 --batch 64 --moves 2

Each arm warms up with one move (every shape its timed window uses), then times --moves moves: a move at N = 400 on the
128-channel CUDA-core towers takes seconds.  Prints one JSON line per board side and a last line with the card's name
and power limit.  The weights are synthetic (seed 0): the rate does not depend on them."""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def kernel_shares(cfg, weights, B):
    """{kernel class: ms} of one search of B empty boards with every kernel bracketed by events."""
    import numpy
    from muzero_general_b200.engine import SearchEngine
    eng = SearchEngine(cfg, max_games=B, num_simulations=cfg.num_simulations)
    eng.load_weights(weights)
    obs = numpy.zeros((B,) + tuple(cfg.observation_shape), numpy.float32)
    obs[:, 2] = 1.0
    eng.search(obs=obs, add_exploration_noise=True)                  # warm-up, untimed
    eng.kernel_timing(True)
    eng.kernel_times()
    eng.search(obs=obs, add_exploration_noise=True)
    times = {k: round(ms, 3) for k, (ms, n) in eng.kernel_times().items() if n}
    eng.kernel_timing(False)
    eng.close()
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sides", default="11,15")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--sims", type=int, default=0, help="num_simulations (0: the config's 400)")
    ap.add_argument("--moves", type=int, default=3, help="timed moves of each arm")
    args = ap.parse_args()

    from device_games_rate import card, rate
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    mod = load_game_module("gomoku")
    for side in (int(s) for s in args.sides.split(",")):
        out = {"game": "gomoku", "board_size": side, "actions": side * side, "batch": args.batch}
        for arm, device_envs in (("device", True), ("host", False)):
            cfg = mod.MuZeroConfig(board_size=side)
            cfg.rng_mode, cfg.num_parallel_games = "philox", args.batch
            cfg.num_simulations = args.sims or cfg.num_simulations
            out["num_simulations"] = cfg.num_simulations
            weights = synthetic_weights(netspec_from_config(cfg), 0)
            r, steps, dt = rate(types.SimpleNamespace(Game=mod.Game.sized(side)), cfg, weights, device_envs, 1, args.moves, 0.0)
            out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 2), steps, round(dt, 3)
        out["speedup"] = round(out["device_env_steps_per_s"] / out["host_env_steps_per_s"], 2)
        out["search_kernel_ms"] = kernel_shares(cfg, weights, args.batch)
        total = sum(out["search_kernel_ms"].values())
        out["tree_step_share"] = round(out["search_kernel_ms"].get("tree_step_kernel", 0.0) / total, 4)
        print(json.dumps(out), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
