"""Reanalyse's fresh search rate: Reanalyse.fresh_search on the device route (mz_reanalyse_search: the host hands over
each game's frames once, the GPU builds every stacked input and searches it chunk by chunk) next to the host route (every
position's stack built with GameHistory.get_stacked_observations, then engine.search per chunk with the same chunk
boundaries, legal masks, to_play, game ids and move indices), in one process.

    python scripts/reanalyse_search_rate.py                           # every workload
    python scripts/reanalyse_search_rate.py --workloads connect4_s8

Workloads (synthetic seeded frames and actions, synthetic weights of seed 0, the config's num_simulations unless named):
  tictactoe               TicTacToe (s = 0), 512 games of 9 moves, 1024 positions per chunk
  connect4_s0, _s8        Connect4 at s = 0 and s = 8, 64 games of 42 moves, 1024 positions per chunk
  cartpole                CartPole (the fused FC search), 8 games of 500 moves, 1024 positions per chunk
  atari, atari_wide       games/atari.py (16 x 256 net, s = 32), 4 games of 200 moves, N = 50, 256 positions per chunk,
                          on the CUDA-core towers and on MZ_TC_WIDE=3
Each route first runs the measured games twice (so every chunk shape is warm and the step-wise pipeline's graphs are
captured), then --reps timed runs.  Per workload and route one JSON line: positions/s of the median run (and of the
fastest), the device memory the process holds after the runs (the library's allocations persist, so this is its peak)
and the host peak of one run (tracemalloc, Python allocations), and whether the two routes agree bit for bit in visit
counts and root values; a last line names the card and its power limit."""
import argparse
import json
import os
import sys
import time
import tracemalloc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from reanalyse_rate import _games, card  # noqa: E402

# workload -> (game, s, games, moves, positions per chunk, MZ_TC_WIDE or None)
WORKLOADS = {
    "tictactoe": ("tictactoe", 0, 512, 9, 1024, None),
    "connect4_s0": ("connect4", 0, 64, 42, 1024, None),
    "connect4_s8": ("connect4", 8, 64, 42, 1024, None),
    "cartpole": ("cartpole", 0, 8, 500, 1024, None),
    "atari": ("atari", 32, 4, 200, 256, None),
    "atari_wide": ("atari", 32, 4, 200, 256, "3"),
}


def _host_route(actor, games, ids):
    """Host stacks through engine.search, max_positions positions per call, the same inputs as fresh_search."""
    import numpy
    from muzero_general_b200 import reanalyse as ra
    cfg, eng = actor.config, actor.search_engine
    A, s, B = len(cfg.action_space), cfg.stacked_observations, actor.max_positions
    shape = tuple(cfg.observation_shape)
    flat = [(gh, g, i) for g, gh in enumerate(games) for i in range(len(gh.root_values))]
    visits, root = [], []
    for lo in range(0, len(flat), B):
        part = flat[lo:lo + B]
        obs = numpy.stack([numpy.asarray(gh.get_stacked_observations(i, s, A), numpy.float32).reshape(-1)
                           for gh, _, i in part])
        legal = numpy.concatenate([actor.Game.legal_masks(numpy.asarray(gh.observation_history[i], numpy.float32)
                                                          .reshape((1,) + shape)) for gh, _, i in part])
        out = eng.search(obs=obs, legal_mask=legal, to_play=numpy.array([gh.to_play_history[i] for gh, _, i in part], numpy.int32),
                         add_exploration_noise=True,
                         game_id=numpy.array([ra.Reanalyse.SEARCH_GAME_IDS + ids[g] for _, g, _ in part], numpy.int64),
                         move_index=numpy.array([i for _, _, i in part], numpy.int32))
        visits.append(out.visit_counts)
        root.append(out.root_value)
    return numpy.concatenate(visits), numpy.concatenate(root)


def run(name, reps):
    import numpy
    import torch
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    game, s, n, moves, chunk, wide = WORKLOADS[name]
    os.environ.pop("MZ_TC_WIDE", None)
    if wide:
        os.environ["MZ_TC_WIDE"] = wide
    mod = load_game_module(game)
    cfg = mod.MuZeroConfig()
    cfg.stacked_observations, cfg.reanalyse_search = s, True
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info()[0]
    actor = ra.Reanalyse({"weights": synthetic_weights(netspec_from_config(cfg), 0)}, cfg, max_positions=chunk,
                         Game=mod.Game)
    games = _games(cfg, n, moves, 0)
    for gh in games:
        gh.to_play_history = [t % len(cfg.players) for t in range(len(gh.action_history))]
        if game in ("tictactoe", "connect4"):          # empty boards: every action legal for the hook
            gh.observation_history = [o * 0 for o in gh.observation_history]
    ids = list(range(n))
    def device(g, k):
        out = actor.fresh_search(g, k)
        return numpy.concatenate([v for v, _, _ in out]), numpy.concatenate([r for _, r, _ in out])

    routes = [("device", device), ("host", lambda g, k: _host_route(actor, g, k))]
    lines, results = [], {}
    for route, fn in routes:
        cold = actor.search_engine.numerics
        for _ in range(2):                                 # warm-up on the measured chunks: the first run captures
            results[route] = fn(games, ids)                # the full chunks' graph, the second the last chunk's
        towers, times, repeatable = actor.search_engine.numerics, [], True
        for r in range(reps):
            if r == 0:
                tracemalloc.start()
            t0 = time.perf_counter()
            got = fn(games, ids)
            times.append(time.perf_counter() - t0)
            if r == 0:
                _, peak = tracemalloc.get_traced_memory()
                tracemalloc.stop()
            repeatable &= all(numpy.array_equal(a, b) for a, b in zip(got, results[route]))
        torch.cuda.synchronize()
        held = free0 - torch.cuda.mem_get_info()[0]
        med = sorted(times)[len(times) // 2]
        lines.append(dict(workload=f"{name}: {game} s={s}, N={cfg.num_simulations}, {n} games of {moves} moves, "
                                   f"{chunk} positions per chunk, MZ_TC_WIDE={wide or 'unset'}", route=route,
                          positions=n * moves, reps=reps, positions_per_s=round(n * moves / med, 1),
                          best_positions_per_s=round(n * moves / min(times), 1), median_seconds=round(med, 3),
                          device_gib_held=round(held / 2**30, 2), host_peak_gib=round(peak / 2**30, 3),
                          repeatable=repeatable, numerics_cold=cold, numerics=towers, numerics_after=actor.search_engine.numerics))
    lines[0]["equal_to_host_route"] = all(numpy.array_equal(a, b) for a, b in zip(results["device"], results["host"]))
    actor.close()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    for name in args.workloads:
        for line in run(name, args.reps):
            print(json.dumps(line), flush=True)
    gpu, power = card()
    print(json.dumps(dict(gpu=gpu, power_limit=power)))


if __name__ == "__main__":
    main()
