"""Evaluation throughput: test-mode games against the expert on the device (SelfPlay.play_test_games) next to the
reference's one-game-at-a-time test loop (play_game(0, threshold, False, "expert", 0)), in the same process.

    python scripts/eval_rate.py                      # Connect4, 1024 games on 1024 slots, N = 200, default towers
    python scripts/eval_rate.py --games 4096 --host-games 2

Prints one JSON line: games/s and env-steps/s (moves of the returned games, both sides) of play_test_games, the host
loop's games/s and env-steps/s, the summary of the device games, and the card's name and power limit.  The weights are
synthetic (seed 0): the rate does not depend on them, the win rate does."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in q.split(","))
        return name, power
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--game", default="connect4")
    ap.add_argument("--games", type=int, default=1024, help="test games returned by the timed play_test_games call")
    ap.add_argument("--batch", type=int, default=1024, help="num_parallel_games: slots of the device loop")
    ap.add_argument("--sims", type=int, default=200)
    ap.add_argument("--opponent", default="expert")
    ap.add_argument("--host-games", type=int, default=3, help="games of the host play_game loop")
    args = ap.parse_args()

    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    from muzero_general_b200.self_play import SelfPlay

    mod = load_game_module(args.game)
    cfg = mod.MuZeroConfig()
    cfg.num_simulations, cfg.rng_mode, cfg.num_parallel_games = args.sims, "philox", args.batch
    weights = synthetic_weights(netspec_from_config(cfg), 0)

    worker = SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    worker.play_test_games(1, opponent=args.opponent, muzero_player=0)         # warm-up: one game's worth of moves
    t0 = time.perf_counter()
    games, summary = worker.play_test_games(args.games, opponent=args.opponent, muzero_player=0)
    dt = time.perf_counter() - t0
    plies = int(games.lengths().sum())
    worker.close()

    cfg1 = mod.MuZeroConfig()
    cfg1.num_simulations, cfg1.rng_mode, cfg1.num_parallel_games = args.sims, "philox", 1
    host = SelfPlay({"weights": weights}, mod.Game, cfg1, 0)
    host.play_game(0, cfg1.temperature_threshold, False, args.opponent, 0)      # warm-up
    t1 = time.perf_counter()
    host_plies = sum(len(host.play_game(0, cfg1.temperature_threshold, False, args.opponent, 0).action_history) - 1
                     for _ in range(args.host_games))
    dt_host = time.perf_counter() - t1
    host.close()

    name, power = card()
    device_rate = len(games) / dt
    host_rate = args.host_games / dt_host
    print(json.dumps(dict(
        workload=f"{args.game} vs {args.opponent}, {args.games} games on {args.batch} slots, N={args.sims}",
        device_games_per_s=round(device_rate, 2), device_env_steps_per_s=round(plies / dt, 1),
        device_seconds=round(dt, 3), host_games_per_s=round(host_rate, 4), host_env_steps_per_s=round(host_plies / dt_host, 2),
        host_games=args.host_games, speedup=round(device_rate / host_rate, 1), summary=summary, gpu=name,
        power_limit=power)))


if __name__ == "__main__":
    main()
