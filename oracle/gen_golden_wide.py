"""ORACLE support: fixtures for action spaces beyond 128 - Gomoku on 15 x 15 and 16 x 16 - generated FROM THE
UNMODIFIED REFERENCE with the helpers of ``oracle/gen_golden.py``.

Run where the reference exists (``python -m oracle.gen_golden_wide``); the GPU box only sees the committed outputs
under tests/golden/:

* env_gomoku15.json     playouts on the reference's ``Gomoku`` with ``board_size`` set to 15 and to 16 before
                        ``reset()``: per side, a five in a row on each of the four directions ending at the far edge, and
                        a random playout stopped after ``CUT`` moves (a game that only ``max_moves`` ends).  Asserts that
                        games/gomoku.py at the same ``board_size`` agrees step by step.
* mcts_gomoku15.json    traced reference ``MCTS.run`` searches with 225 actions on a synthetic 2 x 16-channel net
                        (both files in the compact, exact encodings of ``oracle/packing.py``: per-action arrays would
                        otherwise make them megabytes)
* MANIFEST_wide.json    the files above, with the reference root and the torch / numpy versions

The reference's ``get_observation`` builds its side-to-move plane with a literal ``(11, 11)``, which cannot be stacked
with the two stone planes of another side.  The reference is not edited: its module is handed a numpy whose ``full``
takes the board's side for that one literal shape, and everything else of ``step`` runs as written.
"""
import json
import os
import types

import numpy
import torch

from oracle.gen_golden import OUT, run_traced_search, to_torch_sd
from oracle.packing import pack_board, pack_floats, pack_subset
from oracle.refload import REFERENCE_ROOT, load_reference, load_reference_game
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

CUT = 30
# (start row, start column, row step, column step): the fifth stone lands on the last row or column
EDGE_LINES = lambda s: ((s - 1, s - 5, 0, 1), (s - 5, s - 1, 1, 0), (s - 5, s - 5, 1, 1), (s - 1 - 4, 4, 1, -1))


def _numpy_with_side(side):
    shim = types.ModuleType("numpy")
    shim.__dict__.update(numpy.__dict__)
    shim.full = lambda shape, *a, **k: numpy.full((side, side) if tuple(shape) == (11, 11) else shape, *a, **k)
    return shim


def _ref_game(ref_mod, side, seed):
    g = ref_mod.Game(seed)
    g.env.board_size = side
    g.env.board_markers = [chr(x) for x in range(ord("A"), ord("A") + side)]
    return g


def _edge_win(side, line):
    """Moves of a game in which player +1 completes `line` with its fifth stone; player -1 plays the top-left corner
    rows, away from the line."""
    y, x, dy, dx = line
    mine = [(y + i * dy) * side + x + i * dx for i in range(5)]
    other = [a for a in range(side * side) if a not in mine][:4]
    return [a for pair in zip(mine, other + [None]) for a in pair if a is not None]


def _playout(ref_mod, my_mod, side, seed, moves=None, rs=None):
    ref, mine = _ref_game(ref_mod, side, seed), my_mod.Game(seed, board_size=side)
    o_r, o_m = ref.reset(), mine.reset()
    assert numpy.array_equal(numpy.asarray(o_r), o_m) and numpy.asarray(o_r).dtype == o_m.dtype
    steps, done = [], False
    for t in range(len(moves) if moves else CUT):
        legal = ref.legal_actions()
        assert legal == mine.legal_actions() and ref.to_play() == mine.to_play()
        a = int(moves[t]) if moves else int(legal[rs.randint(len(legal))])
        o_r, r_r, done = ref.step(a)
        o_m, r_m, d_m = mine.step(a)
        assert numpy.array_equal(numpy.asarray(o_r), o_m) and r_r == r_m and done == d_m, (side, seed, a)
        assert ref.action_to_string(a) == mine.action_to_string(a)
        steps.append(dict(action=a, reward=int(r_r), done=bool(done), to_play=int(ref.to_play()),
                          legal=pack_subset([int(x) for x in ref.legal_actions()], side * side), obs=pack_board(o_r)))
        if done:
            break
    assert done == bool(moves), "an edge line ends its game on its last move; the random playout is cut before an end"
    return steps


def _pack_search(run):
    assert run["root_actions"] == run["legal"]
    del run["root_actions"]
    A = int(numpy.prod(run["obs_shape"][1:]))
    run["legal"] = pack_subset(run["legal"], A)
    run["root_visits"] = {"n": len(run["root_visits"]), "nonzero": {str(i): v for i, v in enumerate(run["root_visits"]) if v}}
    for key in ("obs", "root_priors_raw", "noise", "root_priors", "root_child_value_sums"):
        run[key] = pack_floats(run[key])
    for sim in run["sims"]:
        sim["priors"] = pack_floats(sim["priors"])
    return run


def main():
    sp, models, replay_buffer, trainer = load_reference()
    import muzero_general_b200.games as mygames
    ref_mod = load_reference_game("gomoku")
    my_mod = mygames.load_game_module("gomoku")
    real_numpy = ref_mod.numpy
    sides = {}
    try:
        for side in (15, 16):
            ref_mod.numpy = _numpy_with_side(side)
            games = [_playout(ref_mod, my_mod, side, k, moves=_edge_win(side, line)) for k, line in enumerate(EDGE_LINES(side))]
            games.append(_playout(ref_mod, my_mod, side, 9, rs=numpy.random.RandomState(31 + side)))
            sides[str(side)] = games
        json.dump(dict(name="gomoku", cut=CUT, sides=sides), open(os.path.join(OUT, "env_gomoku15.json"), "w"))

        # searches with 225 actions: the reference's config with the fields a 15 x 15 board changes, on a small net
        side = 15
        ref_mod.numpy = _numpy_with_side(side)
        ref_cfg = ref_mod.MuZeroConfig()
        ref_cfg.observation_shape = (3, side, side)
        ref_cfg.action_space = list(range(side * side))
        ref_cfg.blocks, ref_cfg.channels = 2, 16
        my_cfg = my_mod.MuZeroConfig(board_size=side)
        my_cfg.blocks, my_cfg.channels = 2, 16
        spec = netspec_from_config(my_cfg)
        net = models.MuZeroNetwork(ref_cfg)
        net.set_weights(to_torch_sd(synthetic_weights(spec, 0)))
        net.eval()
        runs = []
        for moves, n_sim, seed in (((), 8, 0), ((112, 224, 0), 16, 1)):
            ref_cfg.num_simulations = n_sim
            g = _ref_game(ref_mod, side, seed)
            o = g.reset()
            for a in moves:
                o, _, _ = g.step(a)
            runs.append(run_traced_search(sp, ref_cfg, net, o, g.legal_actions(), g.to_play(), True, seed))
        shown = [(max(r["root_visits"]), r["first_index"]) for r in runs]
        json.dump([_pack_search(r) for r in runs], open(os.path.join(OUT, "mcts_gomoku15.json"), "w"))
    finally:
        ref_mod.numpy = real_numpy
    manifest = {"reference_root": REFERENCE_ROOT, "torch": torch.__version__, "numpy": numpy.__version__,
                "files": ["env_gomoku15.json", "mcts_gomoku15.json"]}
    json.dump(manifest, open(os.path.join(OUT, "MANIFEST_wide.json"), "w"), indent=1)
    print("wide fixtures written; (largest root visit count, first-simulation pick):", shown)


if __name__ == "__main__":
    main()
