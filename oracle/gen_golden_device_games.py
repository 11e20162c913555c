"""ORACLE support: fixtures of the two one-player plug-ins that need no third-party package, games/twentyone.py and
games/simple_grid.py, generated FROM THE UNMODIFIED REFERENCE with the helpers of ``oracle/gen_golden.py``.

Run here (``python -m oracle.gen_golden_device_games``), where the reference exists; the GPU box only sees the
committed outputs under tests/golden/:

* env_<game>.json     random playouts on the reference environment; asserts our plug-in agrees step by step
* net_<game>.npz      the reference network on synthetic weights (a 32-channel residual net on a 3x3 board, an FC
                      net with encoding 5)
* mcts_<game>.json    traced reference searches
* MANIFEST_device_games.json   the files above, with the reference root and the torch / numpy versions

It also asserts that each plug-in's config and weights_spec agree with the reference's.
"""
import json
import os

import numpy
import torch

from oracle.gen_golden import OUT, check_config_and_spec, gen_env_fixture, gen_net, run_traced_search
from oracle.refload import REFERENCE_ROOT, load_reference, load_reference_game
from muzero_general_b200.netspec import synthetic_weights

# game -> (playouts, network batch, search starts: (moves from reset, num_simulations, seed))
GAMES = {
    "twentyone": (24, 8, (((), 21, 0), ((0,), 50, 1), ((0, 0), 50, 2))),
    "simple_grid": (8, 8, (((), 10, 0), ((1,), 30, 1), ((0, 1, 1), 30, 2))),
}


def main():
    sp, models, replay_buffer, trainer = load_reference()
    import muzero_general_b200.games as mygames
    written = []
    for name, (n_env, batch, starts) in GAMES.items():
        ref_game = load_reference_game(name)
        my_mod = mygames.load_game_module(name)
        ref_cfg = ref_game.MuZeroConfig()
        spec = check_config_and_spec(models, name, ref_cfg, my_mod.MuZeroConfig())
        fx = gen_env_fixture(ref_game, my_mod, name, n_env, seed=31)
        json.dump(fx, open(os.path.join(OUT, f"env_{name}.json"), "w"))
        net = gen_net(models, name, ref_cfg, spec, synthetic_weights(spec, 0), batch, seed=37)
        runs = []
        for moves, n_sim, seed in starts:
            ref_cfg.num_simulations = n_sim
            g = ref_game.Game(seed)
            o = g.reset()
            for a in moves:
                o, _, _ = g.step(a)
            runs.append(run_traced_search(sp, ref_cfg, net, o, g.legal_actions(), g.to_play(), True, seed))
        json.dump(runs, open(os.path.join(OUT, f"mcts_{name}.json"), "w"))
        written += [f"env_{name}.json", f"net_{name}.npz", f"mcts_{name}.json"]
        print(name, "fixtures written; root visits", [r["root_visits"] for r in runs])
    manifest = {"reference_root": REFERENCE_ROOT, "torch": torch.__version__, "numpy": numpy.__version__, "files": written}
    json.dump(manifest, open(os.path.join(OUT, "MANIFEST_device_games.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
