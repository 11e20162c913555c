"""Test-game rate of host-stepped games: SelfPlay.play_test_games on the device loop with the environment stepped on the
host (config.host_env_device_loop, loop_path "device-host-env") next to the reference's one-game-at-a-time test loop
(play_game(0, threshold, False, opponent, 0), batch-1 searches), in one process.

    python scripts/host_test_games_rate.py                          # every workload
    python scripts/host_test_games_rate.py --workloads connect4_expert --host-games 1

Workloads: Connect4 without its device environment against "expert" and "random" (256 games on 256 slots, N = 50), and
games/atari.py (the 16 x 256 net, stacked_observations = 32, synthetic 3 x 96 x 96 frames) with max_moves cut to 48,
its observations kept on the host (the window layout games/atari.py's full length needs), against "self" (64 games on
64 slots, N = 50).  Each arm warms up first.  Per workload one JSON line: games/s and env-steps/s (moves of the returned
games, both sides) of both arms and their ratio; a last line names the card and its power limit.  The weights are
synthetic (seed 0): the rate does not depend on them, the win rate does."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# workload -> (game, opponent, slots and games, num_simulations, max_moves or None, observations kept on the host)
WORKLOADS = {
    "connect4_expert": ("connect4", "expert", 256, 50, None, False),
    "connect4_random": ("connect4", "random", 256, 50, None, False),
    "atari_48_window": ("atari", "self", 64, 50, 48, True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def _config(mod, B, sims, max_moves):
    cfg = mod.MuZeroConfig()
    cfg.num_simulations, cfg.rng_mode, cfg.num_parallel_games = sims, "philox", B
    cfg.device_envs, cfg.host_env_device_loop = False, True
    if max_moves:
        cfg.max_moves = max_moves
    return cfg


def run(name, host_games):
    from muzero_general_b200 import self_play as sp
    from muzero_general_b200.engine import HostEnvSelfPlayLoop
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    game, opponent, B, sims, max_moves, window = WORKLOADS[name]
    mod = load_game_module(game)
    cfg = _config(mod, B, sims, max_moves)
    weights = synthetic_weights(netspec_from_config(cfg), 0)
    if window:
        sp.HostEnvSelfPlayLoop = lambda *a, obs_history=None, **kw: HostEnvSelfPlayLoop(*a, obs_history="host", **kw)
    worker = sp.SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    assert worker.loop_path == "device-host-env"
    worker.play_test_games(1, opponent=opponent, muzero_player=0)               # warm-up
    t0 = time.perf_counter()
    games, summary = worker.play_test_games(B, opponent=opponent, muzero_player=0)
    dt = time.perf_counter() - t0
    plies = int(games.lengths().sum())
    worker.close()
    sp.HostEnvSelfPlayLoop = HostEnvSelfPlayLoop

    cfg1 = _config(mod, 1, sims, max_moves)
    host = sp.SelfPlay({"weights": weights}, mod.Game, cfg1, 0)
    host.play_game(0, cfg1.temperature_threshold, False, opponent, 0)         # warm-up
    t1 = time.perf_counter()
    host_plies = sum(len(host.play_game(0, cfg1.temperature_threshold, False, opponent, 0).action_history) - 1
                     for _ in range(host_games))
    dt_host = time.perf_counter() - t1
    host.close()
    rate, host_rate = len(games) / dt, host_games / dt_host
    return dict(workload=f"{name}: {game} vs {opponent}, {len(games)} games on {B} slots, N={sims}, "
                         f"max_moves={cfg.max_moves}, observations on the {'host' if window else 'device'}",
                games_per_s=round(rate, 3), env_steps_per_s=round(plies / dt, 1), seconds=round(dt, 2),
                play_game_games_per_s=round(host_rate, 4), play_game_env_steps_per_s=round(host_plies / dt_host, 2),
                play_game_games=host_games, speedup=round(rate / host_rate, 1), summary=summary)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--host-games", type=int, default=2, help="games of the batch-1 play_game loop per workload")
    args = ap.parse_args()
    for name in args.workloads:
        print(json.dumps(run(name, args.host_games)), flush=True)
    gpu, power = card()
    print(json.dumps(dict(gpu=gpu, power_limit=power)))


if __name__ == "__main__":
    main()
