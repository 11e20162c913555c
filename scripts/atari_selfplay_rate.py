"""Self-play rate of games/atari.py as shipped (max_moves = 27000, stacked_observations = 32, the 16 x 256 net, 3 x 96 x 96
synthetic frames) and of Breakout's shipped max_moves = 2500: the device loop for host-stepped games
(config.host_env_device_loop, which keeps the stack's window on the device and the games' observations on the host when
the whole games do not fit) next to the host loop (BatchedSelfPlay) at the same batch, in one process.

    python scripts/atari_selfplay_rate.py                             # every workload
    python scripts/atari_selfplay_rate.py --workloads atari_64_tc3 --moves 4

Workloads: games/atari.py at 64 and 128 slots, N = 50, on the default (CUDA-core) towers and on MZ_TC_WIDE=3; Breakout
(N = 30, no stack) at 256 slots.  Each arm warms up, then plays --moves moves of the whole batch (the synthetic episode
is 64 moves, so these windows contain no game end).  Per workload one JSON line: env-steps/s of both arms, the device
loop's split of a move into device time (library calls, which end in a synchronisation) and host-environment time (step,
reset, legal mask, to_play), who keeps the observations, and the device bytes per slot of the loop (free device memory
before and after it begins, over the slots).  A last line names the card and its power limit.  The weights are
synthetic (seed 0): the rate does not depend on them."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# workload -> (game, num_parallel_games, num_simulations, MZ_TC_WIDE or None)
WORKLOADS = {
    "atari_64": ("atari", 64, 50, None),
    "atari_64_tc3": ("atari", 64, 50, "3"),
    "atari_128": ("atari", 128, 50, None),
    "atari_128_tc3": ("atari", 128, 50, "3"),
    "breakout_2500": ("breakout", 256, 30, None),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def rate(mod, cfg, weights, new_path, warm, moves):
    """One arm: (env-steps/s, env-steps, seconds, {split and memory of the new path})."""
    import torch
    from muzero_general_b200 import self_play as sp
    cfg.host_env_device_loop = new_path
    worker = sp.SelfPlay({"weights": weights}, mod.Game, cfg, 0)
    assert worker.loop_path == ("device-host-env" if new_path else "host")
    extra = {}
    if new_path:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        worker._device_loop = sp.DeviceHostEnvSelfPlay(worker, cfg.temperature_threshold)
        torch.cuda.synchronize()
        extra["device_bytes_per_slot"] = (free0 - torch.cuda.mem_get_info()[0]) // cfg.num_parallel_games
        extra["obs_history"] = worker._device_loop.loop.obs_history
    worker.play_moves(warm, 1.0)
    loop = worker._device_loop
    dev0, env0 = (loop.device_s, loop.env_s) if new_path else (0.0, 0.0)
    start, t0 = worker.env_steps, time.perf_counter()
    for _ in range(moves):
        worker.play_moves(1, 1.0)
    dt = time.perf_counter() - t0
    steps = worker.env_steps - start
    if new_path:
        extra["device_ms_per_move"] = round(1e3 * (loop.device_s - dev0) / moves, 2)
        extra["host_env_ms_per_move"] = round(1e3 * (loop.env_s - env0) / moves, 2)
    worker.close()
    return steps / dt, steps, dt, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--warmup", type=int, default=2, help="moves of the whole batch before the timed ones")
    ap.add_argument("--moves", type=int, default=4, help="timed moves of the whole batch, per arm")
    args = ap.parse_args()

    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    for wl in args.workloads.split(","):
        game, B, N, wide = WORKLOADS[wl]
        if wide:
            os.environ["MZ_TC_WIDE"] = wide
        else:
            os.environ.pop("MZ_TC_WIDE", None)
        mod = load_game_module(game)
        out = {"workload": wl, "batch": B, "num_simulations": N, "tc_wide": wide}
        for arm, new_path in (("host_loop", False), ("device_host_env", True)):
            cfg = mod.MuZeroConfig()
            cfg.rng_mode, cfg.num_parallel_games, cfg.num_simulations = "philox", B, N
            out["max_moves"], out["stacked_observations"] = cfg.max_moves, cfg.stacked_observations
            r, steps, dt, extra = rate(mod, cfg, synthetic_weights(netspec_from_config(cfg), 0), new_path, args.warmup,
                                       args.moves)
            out[f"{arm}_env_steps_per_s"], out[f"{arm}_env_steps"], out[f"{arm}_seconds"] = round(r, 1), steps, round(dt, 3)
            out.update(extra)
        out["speedup"] = round(out["device_host_env_env_steps_per_s"] / out["host_loop_env_steps_per_s"], 2)
        print(json.dumps(out), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
