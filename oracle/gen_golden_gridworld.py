"""ORACLE support: fixtures of games/gridworld.py, generated FROM THE UNMODIFIED REFERENCE with the helpers of
``oracle/gen_golden.py``.

Run here (``python -m oracle.gen_golden_gridworld``), where the reference exists; the GPU box only sees the committed
outputs under tests/golden/.  The reference's ``games/gridworld.py`` imports gym_minigrid, which is not installed: a
stub module stands in for it, and only the reference's ``MuZeroConfig`` is used.  The environment itself has no
reference fixture; searches start from observations of this repository's restatement of its rules.

* config_gridworld.json   the reference config's values and its visit_softmax_temperature_fn at sample steps
* net_gridworld.npz       the reference network (an FC net with encoding 8 on 147 inputs) on synthetic weights
* mcts_gridworld.json     traced reference searches
* MANIFEST_gridworld.json the files above, with the reference root and the torch / numpy versions

It also asserts that the plug-in's config and weights_spec agree with the reference's.
"""
import json
import os
import sys
import types

import numpy
import torch

from oracle.gen_golden import OUT, check_config_and_spec, gen_net, run_traced_search
from oracle.refload import REFERENCE_ROOT, load_reference, load_reference_game
from muzero_general_b200.netspec import synthetic_weights

# search starts: (placement seed, actions from reset, num_simulations, search seed)
STARTS = (
    (0, (), 20, 0),
    (1, (2, 2, 1), 20, 1),
    (2, (0, 2, 2, 2, 2), 40, 2),
    (3, (1, 1, 2), 40, 3),
)
TEMPERATURE_STEPS = (0, 1, 14999, 15000, 22499, 22500, 30000, 10 ** 6)


def config_values(cfg):
    skip = {"results_path", "train_on_gpu"}
    values = {k: (list(v) if isinstance(v, tuple) else v) for k, v in vars(cfg).items() if k not in skip}
    temps = [[s, cfg.visit_softmax_temperature_fn(s)] for s in TEMPERATURE_STEPS]
    return dict(values=values, temperature=temps)


def main():
    sys.modules.setdefault("gym_minigrid", types.ModuleType("gym_minigrid"))
    sp, models, replay_buffer, trainer = load_reference()
    import muzero_general_b200.games as mygames
    name = "gridworld"
    ref_game = load_reference_game(name)
    my_mod = mygames.load_game_module(name)
    ref_cfg = ref_game.MuZeroConfig()
    spec = check_config_and_spec(models, name, ref_cfg, my_mod.MuZeroConfig())
    json.dump(config_values(ref_cfg), open(os.path.join(OUT, f"config_{name}.json"), "w"), indent=1)
    net = gen_net(models, name, ref_cfg, spec, synthetic_weights(spec, 0), 8, seed=43)
    runs = []
    for place_seed, moves, n_sim, seed in STARTS:
        ref_cfg.num_simulations = n_sim
        g = my_mod.Game(place_seed)
        o = g.reset()
        for a in moves:
            o, _, done = g.step(a)
            assert not done
        runs.append(run_traced_search(sp, ref_cfg, net, o, g.legal_actions(), g.to_play(), True, seed))
    json.dump(runs, open(os.path.join(OUT, f"mcts_{name}.json"), "w"))
    written = [f"config_{name}.json", f"net_{name}.npz", f"mcts_{name}.json"]
    print(name, "fixtures written; root visits", [r["root_visits"] for r in runs])
    manifest = {"reference_root": REFERENCE_ROOT, "torch": torch.__version__, "numpy": numpy.__version__, "files": written}
    json.dump(manifest, open(os.path.join(OUT, "MANIFEST_gridworld.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
