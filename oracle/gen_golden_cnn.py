"""ORACLE support: fixtures for ``downsample="CNN"`` (DownsampleCNN, models.py:278-297), generated FROM THE UNMODIFIED
REFERENCE with the helpers of ``oracle/gen_golden.py`` (``python -m oracle.gen_golden_cnn``).  Observations are not
stored: each fixture keeps the numpy legacy seed that draws them (version-stable streams).

* net_breakout_cnn.npz        Breakout with downsample="CNN", synthetic weights: initial and recurrent inference of
                              ``models.MuZeroNetwork`` on ``RandomState(obs_seed)`` frames, the state_dict keys and shapes
* net_cnn_shapes.npz          initial inference of small CNN nets at 3x24x24, 3x96x64, 3x210x160 and a stacked input
                              (s = 4, 19 planes); input = ``RandomState(i).randint(0, 256)`` / 255 in fp32
* cnn_geometry.npz            for (H, W) in 6..112 x 6..112 and 210 x 160: whether DownsampleCNN's forward raises
* mcts_breakout_cnn_n50.json  traced reference ``MCTS.run`` searches, N = 50, on the Breakout-CNN net
"""
import json
import os

import numpy
import torch

from oracle.gen_golden import OUT, check_config_and_spec, run_traced_search, to_torch_sd
from oracle.refload import REFERENCE_ROOT, load_reference, load_reference_game
from muzero_general_b200.netspec import synthetic_weights

# (name, obs (C, H, W), stacked, channels, blocks) of the shapes fixture; small heads keep it small
SHAPES = (("s24", (3, 24, 24), 0, 8, 1), ("s96x64", (3, 96, 64), 0, 8, 1), ("s210", (3, 210, 160), 0, 4, 0),
          ("stack4", (3, 96, 96), 4, 8, 1))
SMALL_HEADS = dict(reduced_channels_reward=2, reduced_channels_value=2, reduced_channels_policy=2,
                   resnet_fc_reward_layers=[8], resnet_fc_value_layers=[8], resnet_fc_policy_layers=[8])


def _net(models, ref_mod, my_mod, name, **over):
    ref_cfg, my_cfg = ref_mod.MuZeroConfig(), my_mod.MuZeroConfig()
    for c in (ref_cfg, my_cfg):
        c.downsample = "CNN"
        for k, v in over.items():
            setattr(c, k, v)
    spec = check_config_and_spec(models, name, ref_cfg, my_cfg)     # also: weights_spec == the reference's state_dict
    net = models.MuZeroNetwork(ref_cfg)
    net.set_weights(to_torch_sd(synthetic_weights(spec, 0)))
    net.eval()
    return ref_cfg, spec, net


def main():
    torch.set_num_threads(1)
    sp, models, _, _ = load_reference()
    import muzero_general_b200.games as mygames
    ref_mod, my_mod = load_reference_game("breakout"), mygames.load_game_module("breakout")
    s = lambda t: models.support_to_scalar(t, 10).numpy()[:, 0]

    ref_cfg, spec, net = _net(models, ref_mod, my_mod, "breakout_cnn")
    rs = numpy.random.RandomState(3)
    obs = rs.random_sample((2, spec.in_channels) + spec.obs_shape[1:]).astype(numpy.float32)
    act = rs.randint(0, spec.action_space, size=(2, 1)).astype(numpy.int64)
    with torch.no_grad():
        v0, _, p0, h0 = net.initial_inference(torch.from_numpy(obs))
        v1, r1, p1, h1 = net.recurrent_inference(h0, torch.from_numpy(act))
    sd = net.get_weights()
    numpy.savez_compressed(os.path.join(OUT, "net_breakout_cnn.npz"), obs_seed=3, action=act,
                           init_value=v0.numpy(), init_policy=p0.numpy(), init_hidden=h0.numpy(), init_value_scalar=s(v0),
                           rec_value=v1.numpy(), rec_reward=r1.numpy(), rec_policy=p1.numpy(), rec_hidden=h1.numpy(),
                           keys=numpy.array(list(sd)), shapes=numpy.array(json.dumps([list(t.shape) for t in sd.values()])))

    out = {}
    for i, (name, shape, st, ch, blocks) in enumerate(SHAPES):
        _, sp_i, net_i = _net(models, ref_mod, my_mod, name, observation_shape=shape, stacked_observations=st,
                              channels=ch, blocks=blocks, **SMALL_HEADS)
        x = numpy.random.RandomState(i).randint(0, 256, size=(1, sp_i.in_channels) + shape[1:]).astype(numpy.float32)
        with torch.no_grad():
            v, _, p, h = net_i.initial_inference(torch.from_numpy(x / numpy.float32(255)))
        out.update({f"{name}_value": v.numpy(), f"{name}_policy": p.numpy(), f"{name}_hidden": h.numpy()})
    numpy.savez_compressed(os.path.join(OUT, "net_cnn_shapes.npz"), **out)

    def raises(H, W):
        try:
            with torch.no_grad():
                models.DownsampleCNN(3, 4, (-(-H // 16), -(-W // 16)))(torch.zeros(1, 3, H, W))
            return 0
        except RuntimeError:
            return 1
    sizes = numpy.arange(6, 113, dtype=numpy.int32)
    table = numpy.array([[raises(int(H), int(W)) for W in sizes] for H in sizes], numpy.uint8)
    numpy.savez_compressed(os.path.join(OUT, "cnn_geometry.npz"), sizes=sizes, raises=table,
                           extra=numpy.array([[210, 160, raises(210, 160)]], numpy.int32))

    ref_cfg.num_simulations = 50
    runs = []
    for obs_seed, seed in ((19, 5), (23, 6)):
        o = numpy.random.RandomState(obs_seed).random_sample((3, 96, 96)).astype(numpy.float32)
        run = run_traced_search(sp, ref_cfg, net, o, [0, 1, 2, 3], 0, True, seed)
        del run["obs"]
        runs.append(dict(run, obs_seed=obs_seed))
    json.dump(runs, open(os.path.join(OUT, "mcts_breakout_cnn_n50.json"), "w"))
    files = ["net_breakout_cnn.npz", "net_cnn_shapes.npz", "cnn_geometry.npz", "mcts_breakout_cnn_n50.json"]
    json.dump({"reference_root": REFERENCE_ROOT, "torch": torch.__version__, "numpy": numpy.__version__, "files": files},
              open(os.path.join(OUT, "MANIFEST_cnn.json"), "w"), indent=1)
    print(f"{int(table.sum())} of {table.size} geometries raise; root visits:", [r["root_visits"] for r in runs])


if __name__ == "__main__":
    main()
