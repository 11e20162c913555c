"""Self-play rate of games played with their host environments: env-steps/s of SelfPlay.play_moves on the host loop
(BatchedSelfPlay: stacked observations, uploads, sampling and records in Python, one mz_search per move) next to the
device loop for host-stepped games (config.host_env_device_loop: only the environment step on the host) at the same
batch size, in one process, and the new path's split of each move into device time (the library calls, which end in a
synchronisation) and host-environment time (step, reset, legal mask, to_play).

    python scripts/host_env_rate.py                                  # every workload
    python scripts/host_env_rate.py --workloads simple_grid --seconds 10

Workloads: Simple Grid and TicTacToe with device_envs=False at 4096 games; Breakout's synthetic 3 x 96 x 96 frames at 64
games with max_moves = 64 (the synthetic episode's length), without a stack and with the Atari-style
stacked_observations = 32.  Each arm warms up first, then plays moves until --seconds have passed (Breakout: a fixed
number of moves, seconds each on the host loop).  Prints one JSON line per workload and a last line with the card's
name and power limit.  The weights are synthetic (seed 0): the rate does not depend on them."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# workload -> (game, num_parallel_games, num_simulations, config overrides, warm-up moves, timed moves or None)
WORKLOADS = {
    "simple_grid": ("simple_grid", 4096, 10, dict(device_envs=False), 8, None),
    "tictactoe": ("tictactoe", 4096, 25, dict(device_envs=False), 4, None),
    "breakout": ("breakout", 64, 30, dict(max_moves=64), 2, 24),
    "breakout_stack32": ("breakout", 64, 30, dict(max_moves=64, stacked_observations=32), 2, 12),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def rate(mod, cfg, weights, new_path, warm, timed, seconds):
    """(env-steps/s, env-steps timed, seconds, device s, host-env s) of play_moves on one arm (the split: new path)."""
    from muzero_general_b200.self_play import SelfPlay
    cfg.host_env_device_loop = new_path
    worker = SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    assert worker.loop_path == ("device-host-env" if new_path else "host")
    worker.play_moves(warm, 1.0)
    loop = worker._device_loop
    dev0, env0 = (loop.device_s, loop.env_s) if new_path else (0.0, 0.0)
    start, moves, t0 = worker.env_steps, 0, time.perf_counter()
    while (moves < timed) if timed else (time.perf_counter() - t0 < seconds):
        worker.play_moves(1, 1.0)
        moves += 1
    dt = time.perf_counter() - t0
    steps = worker.env_steps - start
    split = (loop.device_s - dev0, loop.env_s - env0) if new_path else (None, None)
    worker.close()
    return steps / dt, steps, dt, moves, split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--seconds", type=float, default=5.0, help="timed window of each arm (Breakout: fixed moves)")
    args = ap.parse_args()

    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    for wl in args.workloads.split(","):
        game, B, N, over, warm, timed = WORKLOADS[wl]
        mod = load_game_module(game)
        out = {"workload": wl, "batch": B, "num_simulations": N}
        for arm, new_path in (("host_loop", False), ("device_host_env", True)):
            cfg = mod.MuZeroConfig()
            cfg.rng_mode, cfg.num_parallel_games, cfg.num_simulations = "philox", B, N
            for k, v in over.items():
                setattr(cfg, k, v)
            r, steps, dt, moves, (dev_s, env_s) = rate(mod, cfg, synthetic_weights(netspec_from_config(cfg), 0), new_path,
                                                       warm, timed, args.seconds)
            out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 1), steps, round(dt, 3)
            if new_path:
                out["device_ms_per_move"] = round(1e3 * dev_s / moves, 3)
                out["host_env_ms_per_move"] = round(1e3 * env_s / moves, 3)
        out["speedup"] = round(out["device_host_env_env_steps_per_s"] / out["host_loop_env_steps_per_s"], 2)
        print(json.dumps(out), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
