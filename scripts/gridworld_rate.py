"""Self-play rate of games/gridworld.py: env-steps/s of SelfPlay.play_moves on three loops at the same batch size and
simulation count, in one process:

* device            the device loop (MZ_ENV_GRIDWORLD: environments, sampling and records on the GPU)
* host_stepped      the device loop with GridworldVector stepped on the host (device_envs = False,
                    host_env_device_loop = True)
* host              the host loop (BatchedSelfPlay: numpy environments, one mz_search per move)

    python scripts/gridworld_rate.py                       # 4096 games at N = 20, 5 s per arm
    python scripts/gridworld_rate.py --batch 1024 --seconds 10

Each arm warms up first (every shape its timed window uses), then plays moves until --seconds have passed.  Prints one
JSON line with the three rates and the card's name and power limit, read in the same run.  The weights are synthetic
(seed 0): the rate does not depend on them."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# arm -> (device_envs, host_env_device_loop, loop_path)
ARMS = {"device": (True, False, "device"), "host_stepped": (False, True, "device-host-env"),
        "host": (False, False, "host")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def rate(mod, cfg, weights, arm, warm, seconds):
    """(env-steps/s, env-steps timed, seconds) of play_moves on one arm."""
    from muzero_general_b200.self_play import SelfPlay
    cfg.device_envs, cfg.host_env_device_loop, path = ARMS[arm]
    worker = SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    assert worker.loop_path == path
    worker.play_moves(warm, 1.0)
    start, t0 = worker.env_steps, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        worker.play_moves(4 if arm == "device" else 1, 1.0)
    dt = time.perf_counter() - t0
    steps = worker.env_steps - start
    worker.close()
    return steps / dt, steps, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096, help="num_parallel_games of every arm")
    ap.add_argument("--simulations", type=int, default=20, help="num_simulations (the config's is 20)")
    ap.add_argument("--seconds", type=float, default=5.0, help="timed window of each arm")
    ap.add_argument("--warmup", type=int, default=8, help="moves before each timed window")
    args = ap.parse_args()

    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    mod = load_game_module("gridworld")
    out = {"game": "gridworld", "batch": args.batch, "num_simulations": args.simulations}
    for arm in ARMS:
        cfg = mod.MuZeroConfig()
        cfg.rng_mode, cfg.num_parallel_games, cfg.num_simulations = "philox", args.batch, args.simulations
        r, steps, dt = rate(mod, cfg, synthetic_weights(netspec_from_config(cfg), 0), arm, args.warmup, args.seconds)
        out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 1), steps, round(dt, 3)
    out["card"], out["power_limit"] = name, power
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
