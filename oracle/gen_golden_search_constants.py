"""ORACLE support: reference searches at search constants no shipped game uses, generated FROM THE UNMODIFIED REFERENCE
with the helpers of ``oracle/gen_golden.py``.

Run here (``python -m oracle.gen_golden_search_constants``), where the reference exists; the GPU box only sees the
committed outputs under tests/golden/.  Only the reference config's search constants change (discount, pb_c_base,
pb_c_init, root_exploration_fraction); the networks are the reference's on ``synthetic_weights(spec, 0)`` with the last
layer of the reward head made antisymmetric about the support's centre (``reward_signed_weights``), so that the
predicted rewards take both signs and reach the tree with weight.

* mcts_constants.json.gz     {set id: {game: [traced reference searches]}}, plus "override": {set id: an override_root_with
                             case} (subtree reuse, self_play.py:275-277) on TicTacToe at K1 and K3; gzip-compressed JSON
* MANIFEST_constants.json    the fixture's sha256, the reference root and the torch / numpy versions

For every game and set it asserts that the traces hold predicted rewards of both signs.  They hold no exact tie after
the first simulation: the reference breaks such a tie with numpy.random.choice, which the device and the C oracle do not
restate (they draw from Philox), so a tied trace could only be replayed by oracle/mcts.py.  Ties and paths at least as deep
as a lane group at these constants come from the synthetic teachers of tests/test_search_constants_*.py instead, which
assert both.  Existing fixtures are untouched.
"""
import copy
import gzip
import hashlib
import json
import os

import numpy
import torch

from oracle.gen_golden import OUT, Tracer, board_obs, check_config_and_spec, run_traced_search, to_torch_sd
from oracle.refload import REFERENCE_ROOT, load_reference, load_reference_game
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

FIXTURE = "mcts_constants.json.gz"
# id -> (discount, pb_c_base, pb_c_init, root_exploration_fraction, games)
CONSTANTS = {
    "K1": (0.9, 19652, 1.25, 0.25, ("tictactoe", "connect4", "cartpole")),
    "K2": (0.5, 5, 0.5, 0.0, ("tictactoe", "connect4", "cartpole")),
    "K3": (0.997, 1e6, 3.0, 1.0, ("tictactoe", "cartpole")),
    "K4": (0.0, 50, 1.25, 0.25, ("tictactoe",)),
}
# the override_root_with cases: the default root exploration fraction, and all noise (a continued search mixes it again)
OVERRIDE_KEYS = ("K1", "K3")
# reward head's last layer: (gain on the upper half of the support, logit offset of each half); see reward_signed_weights
REWARD_HEAD = {"tictactoe": (2.0, 0.0), "connect4": (1.0, 0.25), "cartpole": (2.0, 0.0)}
REWARD_LAST = {"tictactoe": "dynamics_network.module.fc.2", "connect4": "dynamics_network.module.fc.2",
               "cartpole": "dynamics_reward_network.module.2"}
# search starts per game: (moves from reset or a CartPole observation, num_simulations, seed)
STARTS = {
    "tictactoe": (((), 30, 0), ((4, 0, 8), 50, 1)),
    "connect4": (((), 30, 0), ((3, 3, 2, 4, 3, 3), 50, 1)),
    "cartpole": (((0.01, -0.02, 0.03, 0.04), 30, 0), ((-0.03, 0.01, 0.02, -0.04), 50, 1)),
}


def apply_constants(cfg, key):
    cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction = CONSTANTS[key][:4]


def reward_signed_weights(name, spec):
    """synthetic_weights(spec, 0) with the reward head's last layer antisymmetric about the support's centre S: row S + k
    scaled by the gain, row S - k its negation, biases -b above the centre and +b below.  Bin S + k and bin S - k then get
    opposite logits, so the sign of a predicted reward follows the hidden state instead of the synthetic biases."""
    gain, b = REWARD_HEAD[name]
    S = spec.support_size
    w = synthetic_weights(spec, 0)
    W = w[f"{REWARD_LAST[name]}.weight"] * numpy.float32(gain)
    W[:S] = -W[S + 1:][::-1]
    bias = numpy.zeros(2 * S + 1, numpy.float32)
    bias[S + 1:], bias[:S] = -b, b
    w[f"{REWARD_LAST[name]}.weight"], w[f"{REWARD_LAST[name]}.bias"] = W.astype(numpy.float32), bias
    return w


def start_obs(ref_game, name, start):
    if name == "cartpole":
        return numpy.array([[start]], dtype=numpy.float32), [0, 1], 0
    return board_obs(ref_game, start)


def check_coverage(key, name, runs):
    rewards = [s["reward"] for r in runs for s in r["sims"]]
    assert min(rewards) < 0 < max(rewards), (key, name, "rewards of one sign only")
    assert all(r["later_ties"] == 0 for r in runs), (key, name, "a tie only numpy's stream can replay")


def override_case(sp, models, ref_game, ref_cfg, net, moves):
    """gen_golden.py's subtree-reuse override_root_with case at this config's constants."""
    o, legal, tp = board_obs(ref_game, moves)
    first = run_traced_search(sp, ref_cfg, net, o, legal, tp, True, 0)
    numpy.random.seed(0)
    with torch.no_grad():
        root, _ = sp.MCTS(ref_cfg).run(net, o, legal, tp, True)
        action = int(sp.SelfPlay.select_action(root, 0))
        ntp = ref_cfg.players[tp + 1] if tp + 1 < len(ref_cfg.players) else ref_cfg.players[0]
        node = root.children[action]
        pre_visits = int(node.visit_count)
        with Tracer(sp) as tr:
            root2, info2 = sp.MCTS(ref_cfg).run(net, None, ref_cfg.action_space, ntp, True, node)
    kids = list(root2.children.keys())
    case = dict(kind="subtree", action=action, to_play=int(ntp), pre_visits=pre_visits,
                noise=tr.dirichlet[0], choices=[[n, i] for n, i in tr.choices],
                root_actions=[int(a) for a in kids],
                root_visits=[int(root2.children[a].visit_count) for a in kids],
                root_child_value_sums=[float(root2.children[a].value_sum) for a in kids],
                root_priors=[float(root2.children[a].prior) for a in kids],
                root_visit_count=int(root2.visit_count), root_value=float(root2.value()),
                max_tree_depth=int(info2["max_tree_depth"]),
                root_predicted_value=info2["root_predicted_value"])
    return dict(first=first, cases=[case])


def main():
    sp, models, replay_buffer, trainer = load_reference()
    import muzero_general_b200.games as mygames
    ref_games, base_cfgs, nets = {}, {}, {}
    for name in ("tictactoe", "connect4", "cartpole"):
        ref_games[name] = load_reference_game(name)
        base_cfgs[name] = ref_games[name].MuZeroConfig()
        spec = check_config_and_spec(models, name, base_cfgs[name], mygames.load_game_module(name).MuZeroConfig())
        net = models.MuZeroNetwork(base_cfgs[name])
        net.set_weights(to_torch_sd(reward_signed_weights(name, spec)))
        net.eval()
        nets[name] = net
    out = {}
    for key, (*_, games) in CONSTANTS.items():
        out[key] = {}
        for name in games:
            cfg = copy.copy(base_cfgs[name])
            apply_constants(cfg, key)
            runs = []
            for start, n_sim, seed in STARTS[name]:
                cfg.num_simulations = n_sim
                o, legal, tp = start_obs(ref_games[name], name, start)
                runs.append(run_traced_search(sp, cfg, nets[name], o, legal, tp, True, seed))
            check_coverage(key, name, runs)
            out[key][name] = runs
            print(key, name, "max depths", [r["max_tree_depth"] for r in runs], "later ties",
                  [r["later_ties"] for r in runs])
    out["override"] = {}
    for key in OVERRIDE_KEYS:
        cfg = copy.copy(base_cfgs["tictactoe"])
        apply_constants(cfg, key)
        cfg.num_simulations = 25
        out["override"][key] = override_case(sp, models, ref_games["tictactoe"], cfg, nets["tictactoe"], (4, 0))
        print(f"override_root_with at {key}:", out["override"][key]["cases"][0]["root_visits"])
    data = gzip.compress(json.dumps(out).encode(), mtime=0)         # mtime 0: regenerated bytes are identical
    with open(os.path.join(OUT, FIXTURE), "wb") as f:
        f.write(data)
    manifest = {"reference_root": REFERENCE_ROOT, "torch": torch.__version__, "numpy": numpy.__version__,
                "files": {FIXTURE: hashlib.sha256(data).hexdigest()}}
    json.dump(manifest, open(os.path.join(OUT, "MANIFEST_constants.json"), "w"), indent=1)


def load_fixture(directory=OUT):
    """The searches of mcts_constants.json.gz, as main() wrote them."""
    with gzip.open(os.path.join(directory, FIXTURE), "rt") as f:
        return json.load(f)


if __name__ == "__main__":
    main()
