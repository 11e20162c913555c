"""ORACLE support: fixtures for Gomoku's own 6 x 128 net on 15 x 15 and 16 x 16 boards - the shapes the 128-channel towers
run on CTA pairs (MZ_TC_WIDE=2) - generated FROM THE UNMODIFIED REFERENCE with the helpers of ``oracle/gen_golden.py`` and
``oracle/gen_golden_wide.py``.

Run where the reference exists (``python -m oracle.gen_golden_gomoku_pair``); the GPU box only sees the committed outputs
under tests/golden/:

* net_gomoku15.npz / net_gomoku16.npz   the reference's ``initial_inference`` and two ``recurrent_inference`` calls on a
                                        few boards (the fields of net_gomoku.npz), synthetic weights seed 0
* mcts_gomoku15_c128.json               two traced reference ``MCTS.run`` searches with 225 actions on the same 15 x 15
                                        net, N = 50, in the packed format of mcts_gomoku15.json
* MANIFEST_gomoku_pair.json             the files above, with the reference root and the torch / numpy versions

As in gen_golden_wide.py the reference's module is handed a numpy whose ``full`` takes the board's side for the one literal
``(11, 11)`` of ``get_observation``; nothing of the reference is edited.
"""
import json
import os

import numpy
import torch

from oracle.gen_golden import OUT, run_traced_search, to_torch_sd
from oracle.gen_golden_wide import _numpy_with_side, _pack_search, _ref_game
from oracle.refload import REFERENCE_ROOT, load_reference, load_reference_game
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights

BATCH = 3
N_SIM = 50


def _ref_config(ref_mod, side):
    cfg = ref_mod.MuZeroConfig()
    cfg.observation_shape = (3, side, side)
    cfg.action_space = list(range(side * side))
    return cfg


def _net_fixture(models, ref_cfg, spec, net, side, seed):
    """net_gomoku.npz's fields for `side`: board-like observations (stones 0 / 1, the side-to-move plane +-1)."""
    rs = numpy.random.RandomState(seed)
    obs = rs.randint(0, 2, size=(BATCH, spec.in_channels) + spec.obs_shape[1:]).astype(numpy.float32)
    obs[:, -1] = rs.choice([-1.0, 1.0], size=(BATCH, 1, 1))
    act = rs.randint(0, spec.action_space, size=(BATCH, 1)).astype(numpy.int64)
    with torch.no_grad():
        v0, r0, p0, h0 = net.initial_inference(torch.from_numpy(obs))
        v1, r1, p1, h1 = net.recurrent_inference(h0, torch.from_numpy(act))
        v2, r2, p2, h2 = net.recurrent_inference(h1, torch.from_numpy((act + 1) % spec.action_space))
        s = lambda t: models.support_to_scalar(t, ref_cfg.support_size).numpy()[:, 0]
        out = dict(obs=obs, action=act,
                   init_value=v0.numpy(), init_policy=p0.numpy(), init_hidden=h0.numpy(),
                   init_value_scalar=s(v0), init_reward_scalar=s(r0),
                   rec_value=v1.numpy(), rec_reward=r1.numpy(), rec_policy=p1.numpy(), rec_hidden=h1.numpy(),
                   rec_value_scalar=s(v1), rec_reward_scalar=s(r1),
                   rec2_value=v2.numpy(), rec2_reward=r2.numpy(), rec2_policy=p2.numpy(), rec2_hidden=h2.numpy())
    name = f"net_gomoku{side}.npz"
    numpy.savez_compressed(os.path.join(OUT, name), **out)
    return name


def main():
    sp, models, replay_buffer, trainer = load_reference()
    import muzero_general_b200.games as mygames
    ref_mod = load_reference_game("gomoku")
    my_mod = mygames.load_game_module("gomoku")
    real_numpy = ref_mod.numpy
    files, shown = [], []
    try:
        for side in (15, 16):
            ref_mod.numpy = _numpy_with_side(side)
            ref_cfg = _ref_config(ref_mod, side)
            my_cfg = my_mod.MuZeroConfig(board_size=side)
            assert (ref_cfg.blocks, ref_cfg.channels) == (my_cfg.blocks, my_cfg.channels) == (6, 128)
            spec = netspec_from_config(my_cfg)
            net = models.MuZeroNetwork(ref_cfg)
            net.set_weights(to_torch_sd(synthetic_weights(spec, 0)))
            net.eval()
            files.append(_net_fixture(models, ref_cfg, spec, net, side, seed=40 + side))
            if side != 15:
                continue
            runs = []
            for moves, seed in (((), 0), ((112, 224, 0), 1)):
                ref_cfg.num_simulations = N_SIM
                g = _ref_game(ref_mod, side, seed)
                o = g.reset()
                for a in moves:
                    o, _, _ = g.step(a)
                runs.append(run_traced_search(sp, ref_cfg, net, o, g.legal_actions(), g.to_play(), True, seed))
            shown = [(max(r["root_visits"]), r["first_index"]) for r in runs]
            json.dump([_pack_search(r) for r in runs], open(os.path.join(OUT, "mcts_gomoku15_c128.json"), "w"))
            files.append("mcts_gomoku15_c128.json")
    finally:
        ref_mod.numpy = real_numpy
    manifest = {"reference_root": REFERENCE_ROOT, "torch": torch.__version__, "numpy": numpy.__version__, "files": files}
    json.dump(manifest, open(os.path.join(OUT, "MANIFEST_gomoku_pair.json"), "w"), indent=1)
    print("gomoku pair fixtures written; (largest root visit count, first-simulation pick):", shown)


if __name__ == "__main__":
    main()
