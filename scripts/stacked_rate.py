"""Self-play rate with stacked observations: env-steps/s of SelfPlay.play_moves on the device loop (the stacked input is
built on the GPU from the game's records) next to the host loop (BatchedSelfPlay: numpy environments and a GameHistory
rebuilt per slot per move for the stack) at stacked_observations 0 and 8, same batch, one process.

    python scripts/stacked_rate.py                            # Connect4 and TicTacToe at their default sizes
    python scripts/stacked_rate.py --games connect4 --stacked 0,8 --seconds 10

Connect4 plays 1024 games at N = 200 on its default towers, TicTacToe 8192 games at N = 50.  Each arm warms up first
(every shape its timed window uses), then plays moves until --seconds have passed (at least two calls).  Prints one JSON
line per (game, stacked_observations) and a last line with the card's name and power limit.  The weights are synthetic
(seed 0): the rate does not depend on them."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from device_games_rate import card  # noqa: E402

# game -> (num_parallel_games, num_simulations, warm-up moves, moves per call)
SIZES = {"connect4": (1024, 200, 2, 4), "tictactoe": (8192, 50, 2, 4)}


def rate(mod, cfg, weights, device_envs, warm, per_call, seconds):
    """(env-steps/s, env-steps timed, seconds) of play_moves on one arm."""
    from muzero_general_b200.self_play import SelfPlay
    cfg.device_envs = device_envs
    worker = SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    assert worker.loop_path == ("device" if device_envs else "host")
    worker.play_moves(warm, 1.0)
    start, calls, t0 = worker.env_steps, 0, time.perf_counter()
    while calls < 2 or time.perf_counter() - t0 < seconds:
        worker.play_moves(per_call, 1.0)
        calls += 1
    dt = time.perf_counter() - t0
    steps = worker.env_steps - start
    worker.close()
    return steps / dt, steps, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", default="connect4,tictactoe")
    ap.add_argument("--stacked", default="0,8", help="stacked_observations values")
    ap.add_argument("--seconds", type=float, default=5.0, help="timed window of each arm")
    args = ap.parse_args()

    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    for game in args.games.split(","):
        B, N, warm, per_call = SIZES[game]
        mod = load_game_module(game)
        for s in (int(x) for x in args.stacked.split(",")):
            out = {"game": game, "batch": B, "num_simulations": N, "stacked_observations": s}
            for arm, device_envs in (("device", True), ("host", False)):
                cfg = mod.MuZeroConfig()
                cfg.rng_mode, cfg.num_parallel_games, cfg.num_simulations, cfg.stacked_observations = "philox", B, N, s
                r, steps, dt = rate(mod, cfg, synthetic_weights(netspec_from_config(cfg), 0), device_envs, warm,
                                    per_call, args.seconds)
                out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 1), steps, round(dt, 3)
            out["speedup"] = round(out["device_env_steps_per_s"] / out["host_env_steps_per_s"], 2)
            print(json.dumps(out), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
