"""Self-play rate of user environments: env-steps/s of SelfPlay.play_moves for Simple Grid and Gridworld on three loops
at the same batch size and simulation count, in one process:

* device            the built-in device environment (MZ_ENV_SIMPLE_GRID / MZ_ENV_GRIDWORLD)
* user_source       the same rules as a user environment (tests/user_env_sources.py as Game.DEVICE_SOURCE,
                    mz_selfplay_begin_user: compiled with NVRTC, stepped and reset on the device)
* host_stepped      the device loop with the game's vector stepped on the host (device_envs = False,
                    host_env_device_loop = True)

    python scripts/user_env_rate.py                        # 4096 games at each game's num_simulations, 5 s per arm
    python scripts/user_env_rate.py --batch 1024 --seconds 10

Each arm warms up first (every shape its timed window uses; the user arm's NVRTC compile happens in its first call and
is reported as compile_s), then plays moves until --seconds have passed.  Prints one JSON line per game with the three
rates and the card's name and power limit, read in the same run.  The weights are synthetic (seed 0)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ARMS = ("device", "user_source", "host_stepped")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def rate(name, mod, cfg, weights, arm, warm, seconds):
    """(env-steps/s, env-steps timed, seconds, seconds of the first call) of play_moves on one arm."""
    from muzero_general_b200.self_play import SelfPlay
    from user_env_sources import SOURCES
    Game = mod.Game
    if arm == "user_source":
        source, state_bytes, _ = SOURCES[name]
        Game = type("UserGame", (mod.Game,), dict(DEVICE_ENV=None, DEVICE_SOURCE=source, DEVICE_STATE_BYTES=state_bytes))
    cfg.device_envs, cfg.host_env_device_loop = arm != "host_stepped", arm == "host_stepped"
    worker = SelfPlay({"weights": weights}, Game, cfg, 0)
    assert worker.loop_path == {"device": "device", "user_source": "device-user-env", "host_stepped": "device-host-env"}[arm]
    t0 = time.perf_counter()
    worker.play_moves(1, 1.0)
    first = time.perf_counter() - t0
    worker.play_moves(warm, 1.0)
    start, t0 = worker.env_steps, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        worker.play_moves(1 if arm == "host_stepped" else 4, 1.0)
    dt = time.perf_counter() - t0
    steps = worker.env_steps - start
    worker.close()
    return steps / dt, steps, dt, first


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", default="simple_grid,gridworld")
    ap.add_argument("--batch", type=int, default=4096, help="num_parallel_games of every arm")
    ap.add_argument("--simulations", type=int, default=0, help="num_simulations, 0 = the game's config")
    ap.add_argument("--seconds", type=float, default=5.0, help="timed window of each arm")
    ap.add_argument("--warmup", type=int, default=8, help="moves before each timed window")
    args = ap.parse_args()

    from muzero_general_b200.engine import debug_user_env_compile
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    from user_env_sources import SOURCES

    card_name, power = card()
    for name in args.games.split(","):
        mod = load_game_module(name)
        out = {"game": name, "batch": args.batch}
        t0 = time.perf_counter()
        rc, _, info = debug_user_env_compile(SOURCES[name][0])
        out["nvrtc_compile_s"], out["user_kernels"] = round(time.perf_counter() - t0, 3), info
        assert rc == 0
        for arm in ARMS:
            cfg = mod.MuZeroConfig()
            cfg.rng_mode, cfg.num_parallel_games = "philox", args.batch
            if args.simulations:
                cfg.num_simulations = args.simulations
            out["num_simulations"] = cfg.num_simulations
            r, steps, dt, first = rate(name, mod, cfg, synthetic_weights(netspec_from_config(cfg), 0), arm, args.warmup,
                                       args.seconds)
            out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 1), steps, round(dt, 3)
            out[f"{arm}_first_call_s"] = round(first, 3)
        out["card"], out["power_limit"] = card_name, power
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
