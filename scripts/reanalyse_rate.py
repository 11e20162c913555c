"""Reanalyse rate with stacked observations: Reanalyse.fresh_root_values on the device route (mz_reanalyse_values: the
host hands over each game's frames once, the GPU builds every stacked input chunk by chunk) next to the host route it
replaced (every position's stack built with GameHistory.get_stacked_observations and numpy.stack-ed up front, then
mz_initial_inference per chunk), in one process.

    python scripts/reanalyse_rate.py                                  # every workload
    python scripts/reanalyse_rate.py --workloads atari_27000

Workloads (synthetic seeded frames and actions, synthetic weights of seed 0; the rate does not depend on them):
  atari_200, atari_200_wide   games/atari.py (16 x 256 net, s = 32, 3 x 96 x 96 frames), 4 games of 200 moves, 512
                              positions per chunk, on the CUDA-core towers and on MZ_TC_WIDE=3
  atari_27000, _wide          one 27000-move games/atari.py game, the device route only (the host route would need
                              130 GB of stacks)
  connect4                    Connect4 at s = 8, default towers, 64 games of 42 moves, 4096 positions per chunk
  breakout                    Breakout at s = 2, 8 games of 500 moves, 1024 positions per chunk
Per workload and route one JSON line: positions/s, seconds, the device memory the process holds after the call (the
library's allocations persist, so this is its peak) and the host peak (tracemalloc, Python allocations); a last line
names the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time
import tracemalloc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# workload -> (game, s, games, moves, positions per chunk, MZ_TC_WIDE or None, host route too)
WORKLOADS = {
    "atari_200": ("atari", 32, 4, 200, 512, None, True),
    "atari_200_wide": ("atari", 32, 4, 200, 512, "3", True),
    "atari_27000": ("atari", 32, 1, 27000, 512, None, False),
    "atari_27000_wide": ("atari", 32, 1, 27000, 512, "3", False),
    "connect4": ("connect4", 8, 64, 42, 4096, None, True),
    "breakout": ("breakout", 2, 8, 500, 1024, None, True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def _games(cfg, n, moves, seed):
    import numpy
    from muzero_general_b200 import self_play as sp
    rs = numpy.random.RandomState(seed)
    A, shape = len(cfg.action_space), tuple(cfg.observation_shape)
    out = []
    for _ in range(n):
        gh = sp.GameHistory()
        frames = numpy.empty((moves + 1,) + shape, numpy.float32)
        for lo in range(0, moves + 1, 1024):
            frames[lo:lo + 1024] = rs.random_sample((min(1024, moves + 1 - lo),) + shape)
        gh.observation_history = list(frames)
        gh.action_history = [0] + [int(a) for a in rs.randint(0, A, moves)]
        gh.root_values = [0.0] * moves
        out.append(gh)
    return out


def _host_route(actor, games):
    """fresh_root_values as it was: every stack built on the host first."""
    import numpy
    cfg = actor.config
    A = len(cfg.action_space)
    obs = numpy.stack([numpy.asarray(gh.get_stacked_observations(i, cfg.stacked_observations, A), numpy.float32)
                       for gh in games for i in range(len(gh.root_values))]).reshape(-1, actor.engine.obs_elems)
    values = numpy.empty(len(obs), numpy.float32)
    for lo in range(0, len(obs), actor.max_positions):
        values[lo:lo + actor.max_positions] = actor.engine.initial_inference(obs[lo:lo + actor.max_positions])["value"]
    return values


def run(name):
    import numpy
    import torch
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    game, s, n, moves, chunk, wide, with_host = WORKLOADS[name]
    os.environ.pop("MZ_TC_WIDE", None)
    if wide:
        os.environ["MZ_TC_WIDE"] = wide
    cfg = load_game_module(game).MuZeroConfig()
    cfg.stacked_observations = s
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info()[0]
    actor = ra.Reanalyse({"weights": synthetic_weights(netspec_from_config(cfg), 0)}, cfg, max_positions=chunk)
    games = _games(cfg, n, moves, 0)
    warm = _games(cfg, 1, 4, 1)
    routes = [("device", lambda g: numpy.concatenate([numpy.atleast_1d(v) for v in actor.fresh_root_values(g)]))]
    if with_host:
        routes.append(("host", lambda g: _host_route(actor, g)))
    lines, results = [], {}
    for route, fn in routes:
        fn(warm)
        tracemalloc.start()
        t0 = time.perf_counter()
        results[route] = fn(games)
        dt = time.perf_counter() - t0
        _, peak = tracemalloc.get_traced_memory()
        tracemalloc.stop()
        torch.cuda.synchronize()
        held = free0 - torch.cuda.mem_get_info()[0]
        lines.append(dict(workload=f"{name}: {game} s={s}, {n} games of {moves} moves, {chunk} positions per chunk, "
                                   f"MZ_TC_WIDE={wide or 'unset'}", route=route, positions=n * moves,
                          positions_per_s=round(n * moves / dt, 1), seconds=round(dt, 2),
                          device_gib_held=round(held / 2**30, 2), host_peak_gib=round(peak / 2**30, 3)))
    if with_host:
        lines[0]["equal_to_host_route"] = bool(numpy.array_equal(results["device"], results["host"]))
    actor.close()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    args = ap.parse_args()
    for name in args.workloads:
        for line in run(name):
            print(json.dumps(line), flush=True)
    gpu, power = card()
    print(json.dumps(dict(gpu=gpu, power_limit=power)))


if __name__ == "__main__":
    main()
