"""Self-play rate of Gomoku, Twenty-One and Simple Grid: env-steps/s of SelfPlay.play_moves on the device loop
(environments, sampling and records on the GPU) next to the host loop (BatchedSelfPlay: numpy environments, one
mz_search per move) at the same batch size, in one process.

    python scripts/device_games_rate.py                       # all three games at their default sizes
    python scripts/device_games_rate.py --games twentyone --seconds 10

Each arm warms up first (every shape its timed window uses), then plays moves until --seconds have passed; Gomoku at
N = 400 on its 6 x 128-channel towers takes seconds per move, so it times a fixed number of moves instead.  Prints one
JSON line per game and a last line with the card's name and power limit.  The weights are synthetic (seed 0): the rate
does not depend on them."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# game -> (num_parallel_games, warm-up moves, timed moves or None for --seconds)
SIZES = {"simple_grid": (4096, 8, None), "twentyone": (2048, 8, None), "gomoku": (128, 1, 3)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def rate(mod, cfg, weights, device_envs, warm, timed, seconds):
    """(env-steps/s, env-steps timed, seconds) of play_moves on one arm."""
    from muzero_general_b200.self_play import SelfPlay
    cfg.device_envs = device_envs
    worker = SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    assert worker.loop_path == ("device" if device_envs else "host")
    worker.play_moves(warm, 1.0)
    start, moves, t0 = worker.env_steps, 0, time.perf_counter()
    while (moves < timed) if timed else (time.perf_counter() - t0 < seconds):
        worker.play_moves(1 if timed else 4, 1.0)
        moves += 1
    dt = time.perf_counter() - t0
    steps = worker.env_steps - start
    worker.close()
    return steps / dt, steps, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", default="gomoku,twentyone,simple_grid")
    ap.add_argument("--seconds", type=float, default=5.0, help="timed window of each arm (Gomoku: fixed moves)")
    ap.add_argument("--batch", type=int, default=0, help="num_parallel_games for every game (0: per-game default)")
    args = ap.parse_args()

    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    for game in args.games.split(","):
        B, warm, timed = SIZES[game]
        B = args.batch or B
        mod = load_game_module(game)
        out = {"game": game, "batch": B}
        for arm, device_envs in (("device", True), ("host", False)):
            cfg = mod.MuZeroConfig()
            cfg.rng_mode, cfg.num_parallel_games = "philox", B
            out["num_simulations"] = cfg.num_simulations
            r, steps, dt = rate(mod, cfg, synthetic_weights(netspec_from_config(cfg), 0), device_envs, warm, timed,
                                args.seconds)
            out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 1), steps, round(dt, 3)
        out["speedup"] = round(out["device_env_steps_per_s"] / out["host_env_steps_per_s"], 2)
        print(json.dumps(out), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
