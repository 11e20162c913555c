"""Test-game rate of user environments: SelfPlay.play_test_games on the "device-user-env" route (TicTacToe and Connect4
restated as CUDA sources with their expert, tests/user_env_expert_sources.py) next to three baselines in one process: the
built-in device environment ("device"), the host-stepped route ("device-host-env": the game's vector stepped in Python)
and the reference's one-game-at-a-time test loop (play_game(0, threshold, False, "expert", muzero_player), batch-1
searches).

    python scripts/user_env_test_games_rate.py                       # every workload
    python scripts/user_env_test_games_rate.py --games tictactoe --slots 256 --sims 25 --play-games 2

Workloads: each game against "expert" (by default opening: --muzero-player 1), on 256 and 1024 slots, N = 25 and 50,
B games per timed call after a warm-up call.  Per workload one JSON line: games/s of every arm and the user route's ratios to them, and the
user route's idle slot-searches per move: slots in play whose side to move is the opponent's when the search runs (a
new game the opponent opens after the opponent ended the last one), counted with peek over a separate run of one move
per call.  A last line names the card and its power limit.  The weights are synthetic (seed 0): the rate does not
depend on them, the win rate does."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def _worker(game, B, sims, route, weights=None):
    from muzero_general_b200 import self_play as sp
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    from user_env_expert_sources import SOURCES

    mod = load_game_module(game)
    cfg = mod.MuZeroConfig()
    cfg.num_simulations, cfg.rng_mode, cfg.num_parallel_games = sims, "philox", B
    Game = mod.Game
    if route == "device-user-env":
        source, state_bytes, _ = SOURCES[game]
        Game = type("UserGame", (mod.Game,), dict(DEVICE_ENV=None, DEVICE_SOURCE=source, DEVICE_STATE_BYTES=state_bytes))
    elif route == "device-host-env":
        cfg.device_envs, cfg.host_env_device_loop = False, True
    elif route == "host":
        cfg.device_envs = False
    weights = weights or synthetic_weights(netspec_from_config(cfg), 0)
    w = sp.SelfPlay({"weights": weights}, Game, cfg, 0)
    assert w.loop_path == route, (w.loop_path, route)
    return w, cfg, weights


def _rate(game, B, sims, route, mp):
    w, _, _ = _worker(game, B, sims, route)
    w.play_test_games(B, "expert", mp)                                 # warm-up: compile, first launches, graphs
    t0 = time.perf_counter()
    games, _ = w.play_test_games(B, "expert", mp)
    dt = time.perf_counter() - t0
    w.close()
    return len(games) / dt, int(games.lengths().sum()) / dt


def _idle(game, B, sims, moves, mp):
    """Idle slot-searches per move of the user route: slots in play whose side to move is not MuZero's at the search."""
    from muzero_general_b200 import self_play as sp
    w, cfg, _ = _worker(game, B, sims, "device-user-env")
    dev = sp.DeviceBatchedSelfPlay(w, cfg.temperature_threshold, "expert", mp, first_game_id=0)
    idle = 0
    for _ in range(moves):
        idle += int((dev.loop.peek()["to_play"] != mp).sum())
        dev.loop.moves(1, 0.0)
        dev.loop.drain()
    w.close()
    return idle / moves


def _play_game_rate(game, sims, n, mp):
    w, cfg, _ = _worker(game, 1, sims, "host")
    w.play_game(0, cfg.temperature_threshold, False, "expert", mp)   # warm-up
    t0 = time.perf_counter()
    for _ in range(n):
        w.play_game(0, cfg.temperature_threshold, False, "expert", mp)
    dt = time.perf_counter() - t0
    w.close()
    return n / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", nargs="+", default=["tictactoe", "connect4"], choices=["tictactoe", "connect4"])
    ap.add_argument("--slots", nargs="+", type=int, default=[256, 1024])
    ap.add_argument("--sims", nargs="+", type=int, default=[25, 50])
    ap.add_argument("--play-games", type=int, default=2, help="games of the batch-1 play_game loop per workload")
    ap.add_argument("--idle-moves", type=int, default=40, help="moves of the idle-search count per workload")
    ap.add_argument("--muzero-player", type=int, default=1, choices=[0, 1],
                    help="1 (the default): the opponent opens, the case where the user route's searches can idle")
    args = ap.parse_args()
    mp = args.muzero_player
    for game in args.games:
        for sims in args.sims:
            play_game = _play_game_rate(game, sims, args.play_games, mp)
            for B in args.slots:
                user, user_steps = _rate(game, B, sims, "device-user-env", mp)
                device, _ = _rate(game, B, sims, "device", mp)
                host, _ = _rate(game, B, sims, "device-host-env", mp)
                idle = _idle(game, B, sims, args.idle_moves, mp)
                print(json.dumps(dict(
                    workload=f"{game} vs expert, muzero_player {mp}, {B} games on {B} slots, N={sims}",
                    user_games_per_s=round(user, 2), user_env_steps_per_s=round(user_steps, 1),
                    device_games_per_s=round(device, 2), host_env_games_per_s=round(host, 2),
                    play_game_games_per_s=round(play_game, 4), user_over_device=round(user / device, 3),
                    user_over_host_env=round(user / host, 2), user_over_play_game=round(user / play_game, 1),
                    idle_slot_searches_per_move=round(idle, 2), idle_share=round(idle / B, 4))), flush=True)
    gpu, power = card()
    print(json.dumps(dict(gpu=gpu, power_limit=power)))


if __name__ == "__main__":
    main()
