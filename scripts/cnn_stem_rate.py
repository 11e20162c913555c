"""Breakout's net with downsample="CNN" against downsample="resnet": initial-inference boards/s at 128, 1024 and 4096
boards, the kernel split (mz_kernel_timing) of one 1024-board inference, a 128-game N = 50 search.  One JSON line per
stem, then the card's name and power limit read in the same run.  Synthetic weights: the rate does not depend on them."""
import json
import os
import sys
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

from device_games_rate import card  # noqa: E402


def main():
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

    name, power = card()
    for stem in ("CNN", "resnet"):
        cfg = load_game_module("breakout").MuZeroConfig()
        cfg.downsample = stem
        spec = netspec_from_config(cfg)
        w = synthetic_weights(spec, 0)
        obs = numpy.random.RandomState(0).random_sample((4096, spec.obs_elems)).astype(numpy.float32)
        out = {"downsample": stem}
        eng = SearchEngine(cfg, max_games=4096, num_simulations=1)
        eng.load_weights(w)
        for n in (128, 1024, 4096):
            reps = max(3, 8192 // n)
            eng.initial_inference(obs[:n])                     # warm-up
            t0 = time.perf_counter()
            for _ in range(reps):
                eng.initial_inference(obs[:n])
            out[f"init_boards_per_s_{n}"] = round(reps * n / (time.perf_counter() - t0), 1)
        eng.kernel_timing(True)
        eng.kernel_times()
        eng.initial_inference(obs[:1024])
        out["kernel_ms_init_1024"] = {k: round(ms, 4) for k, (ms, cnt) in eng.kernel_times().items() if cnt}
        eng.close()
        eng = SearchEngine(cfg, max_games=128, num_simulations=50)
        eng.load_weights(w)
        eng.search(obs=obs[:128], add_exploration_noise=False)
        t0 = time.perf_counter()
        for _ in range(3):
            eng.search(obs=obs[:128], add_exploration_noise=False)
        out["search_128x50_ms"] = round((time.perf_counter() - t0) / 3 * 1e3, 2)
        eng.close()
        print(json.dumps(out), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
