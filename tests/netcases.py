"""Case table of the network routes: every way a network evaluation can be routed through the kernels, each as a game
config with attributes overridden and the route it is meant to take.  Importable without a GPU.

Routes (``ROUTES``) and the cases that take them:

  FC nets differ only in how a SEARCH evaluates them; initial / recurrent inference of every FC case runs the one FC
  inference kernel (fc_infer.cu), so the three FC routes are told apart by the in-search test (SEARCH_CASES):
  fc_fixed        fused FC search, fully unrolled CartPole shape (E 8, hidden 16, support 10, |A| 2): fc_cartpole
  fc_generic      fused FC search, generic layer walker: fc_e5_a3 (E 5, no representation layer, reward [3, 9],
                  value [], policy [33], |A| 3, support 4), fc_cartpole_s20 (CartPole with support 20)
  fc_stepwise     |A| > 32: step-wise search, 32 lanes striding over the outputs: fc_a40 (|A| 40, E 32, support 300)
  (fixed versus generic is decided by fc_net.cuh::fc_matches_fixed from the shape alone: tests/test_netcases_cpu.py
  checks the shapes; no kernel counter separates the two)
  tc              64-channel tensor-core towers (x3 and fp16): tc_1x1, tc_1x7, tc_6x1, tc_3x3 (narrow P64C4 heads),
                  tc_5x4, tc_6x6, tc_6x7, tc_6x7_a1, tc_6x7_a128, tc_6x7_stack2 (11 input planes), tc_6x7_b0 (no blocks),
                  tc_6x7_b4 (4 blocks: the representation and prediction towers fill one 8-layer launch), tc_6x7_b6 (6
                  blocks: every tower is split across launches)
                  and the edge-weight cases tc_6x7_const, tc_6x7_tiny, tc_5x4_tiny, tc_6x7_wide, tc_6x7_sat,
                  tc_3x3_large / tiny_bn / overflow, tc_5x4_large / tiny_bn / overflow
  tc_heads_left   64 channels whose head weights exceed shared memory: kept off the tensor cores from mz_create on
                  (CUDA-core towers, generic heads), in either tower mode: tc_6x7_bigheads, tc_6x7_s300 (support 300)
  small_tower     fused CUDA-core tower (small_tower.cu): st_c32_6x7, st_16x8_c16, st_1x2, st_c32_const,
                  st_c32_tiny, st_1x2_b0 (no blocks)
  per_layer       one conv3x3 launch per conv: pl_9x9_c32, pl_c48_6x7 (48 channels: no tensor cores, and the weights
                  of a block exceed the fused tower's shared memory), pl_3x3_nofuse (MZ_NO_FUSE=1), pl_9x9_wide,
                  pl_c96_6x7 (96 channels: a full cout tile of 64 and a last one of 32)
  small_search    fused small-network search (small_search.cu): ss_3x3_a2_c8, ss_3x3_a16_c20 (two blocks; with 32
                  channels the weights of two blocks exceed shared memory), ss_5x6_a4, ss_7x3_a12, ss_5x6_tiny
  heads_wide      heads_kernel<128> (C*HW > 1024) on the CUDA-core route: hw_c128_6x7
  heads_big       generic heads route (weights beyond shared memory) on the CUDA-core route: hb_c32_6x7
  downsample      DownSample stem: ds_20x24 (3 x 20 x 24 frames -> 2 x 2 hidden, 16 channels), ds_c96_20x24 (96
                  channels: the stride-2 48 -> 96 conv and the 96-channel blocks have a 32-channel last cout tile),
                  ds_33x17 (every halving of the frame odd), ds_c8_1x1 (C / 2 = 4 channels on a 1 x 1
                  frame), ds_breakout_96x96 (games/breakout.py's net), ds_atari_96x96 (games/atari.py's 131 planes, 256
                  channels and support 300 with the generic heads, one block per tower so the fp64 oracle stays short;
                  batches of 1 to 3) and ds_atari_96x96_wide (the same under MZ_TC_WIDE=3: the towers on the 256-channel
                  x3 tensor-core route, the stem on the CUDA cores)

Edge weights (``edge_weights``), applied to the representation and dynamics towers:

  const   channel c of the hidden state is exactly constant over the board (stem and every conv2 into c zeroed): the
          rescale takes its sc < 1e-5 branch with sc = 0 and the channel must come out exactly 0
  tiny    channel c spans ~1e-6 over the board (conv2 into c zeroed, stem into c x 3e-7): the rescale divides by
          sc + 1e-5, so the value of that epsilon shows
  wide    the last conv of every tower has rows whose largest weight spans 1e-8 ... 1e3, and one all-zero row (per-row
          2^k scaling of the x3 weight image)
  sat     final value / reward FC layers scaled so the logits spread over ~100 (support 300): support_to_scalar near
          its ends
  large / tiny_bn / overflow   netspec.stress_weights
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field

import numpy

from muzero_general_b200.netspec import RESNET, netspec_from_config, stress_weights, synthetic_weights

ROUTES = ("fc_fixed", "fc_generic", "fc_stepwise", "tc", "tc_heads_left", "small_tower", "per_layer", "small_search",
          "heads_wide", "heads_big", "downsample")


@dataclass
class NetCase:
    name: str
    game: str
    route: str
    over: dict = field(default_factory=dict)
    weights: str = "synthetic"          # synthetic | const | tiny | wide | sat | large | tiny_bn | overflow
    env: dict = field(default_factory=dict)
    batches: tuple = ()                 # the inference sweep's batch sizes, when not the route's default

    @property
    def tensor_cores(self):
        return self.route == "tc"


def _board(h, w, a, c=64, blocks=2, **kw):
    return dict(observation_shape=(3, h, w), action_space=list(range(a)), channels=c, blocks=blocks, **kw)


_HEADS16 = dict(reduced_channels_reward=4, reduced_channels_value=4, reduced_channels_policy=4,
                resnet_fc_reward_layers=[16], resnet_fc_value_layers=[16], resnet_fc_policy_layers=[16])

CASES = [
    NetCase("fc_cartpole", "cartpole", "fc_fixed"),
    NetCase("fc_e5_a3", "cartpole", "fc_generic",
            dict(encoding_size=5, fc_representation_layers=[], fc_reward_layers=[3, 9], fc_value_layers=[],
                 fc_policy_layers=[33], action_space=list(range(3)), support_size=4)),
    NetCase("fc_cartpole_s20", "cartpole", "fc_generic", dict(support_size=20)),
    NetCase("fc_a40", "cartpole", "fc_stepwise", dict(action_space=list(range(40)), encoding_size=32, support_size=300)),

    NetCase("tc_1x1", "connect4", "tc", _board(1, 1, 4)),
    NetCase("tc_1x7", "connect4", "tc", _board(1, 7, 7)),
    NetCase("tc_6x1", "connect4", "tc", _board(6, 1, 3)),
    NetCase("tc_3x3", "connect4", "tc", _board(3, 3, 9)),
    NetCase("tc_5x4", "connect4", "tc", _board(5, 4, 6)),
    NetCase("tc_6x6", "connect4", "tc", _board(6, 6, 4)),
    NetCase("tc_6x7", "connect4", "tc"),
    NetCase("tc_6x7_a1", "connect4", "tc", dict(action_space=[0])),
    NetCase("tc_6x7_a128", "connect4", "tc", dict(action_space=list(range(128)))),
    NetCase("tc_6x7_stack2", "connect4", "tc", dict(stacked_observations=2)),
    NetCase("tc_6x7_b0", "connect4", "tc", dict(blocks=0)),
    NetCase("tc_6x7_b4", "connect4", "tc", dict(blocks=4)),
    NetCase("tc_6x7_b6", "connect4", "tc", dict(blocks=6)),
    NetCase("tc_6x7_const", "connect4", "tc", weights="const"),
    NetCase("tc_6x7_tiny", "connect4", "tc", weights="tiny"),
    NetCase("tc_5x4_tiny", "connect4", "tc", _board(5, 4, 6), weights="tiny"),
    NetCase("tc_6x7_wide", "connect4", "tc", weights="wide"),
    NetCase("tc_6x7_sat", "connect4", "tc", dict(support_size=300, resnet_fc_value_layers=[16], resnet_fc_reward_layers=[16]),
            weights="sat"),
    NetCase("tc_3x3_large", "connect4", "tc", _board(3, 3, 9), weights="large"),
    NetCase("tc_3x3_tiny_bn", "connect4", "tc", _board(3, 3, 9), weights="tiny_bn"),
    NetCase("tc_3x3_overflow", "connect4", "tc", _board(3, 3, 9), weights="overflow"),
    NetCase("tc_5x4_large", "connect4", "tc", _board(5, 4, 6), weights="large"),
    NetCase("tc_5x4_tiny_bn", "connect4", "tc", _board(5, 4, 6), weights="tiny_bn"),
    NetCase("tc_5x4_overflow", "connect4", "tc", _board(5, 4, 6), weights="overflow"),
    NetCase("tc_6x7_bigheads", "connect4", "tc_heads_left", dict(reduced_channels_value=16, resnet_fc_value_layers=[128])),
    NetCase("tc_6x7_s300", "connect4", "tc_heads_left", dict(support_size=300)),

    NetCase("st_c32_6x7", "connect4", "small_tower", dict(channels=32, blocks=1)),
    NetCase("st_16x8_c16", "connect4", "small_tower", _board(16, 8, 8, c=16, **_HEADS16)),
    NetCase("st_1x2", "connect4", "small_tower", _board(1, 2, 2, c=16, **_HEADS16)),
    NetCase("st_c32_const", "connect4", "small_tower", dict(channels=32, blocks=1), weights="const"),
    NetCase("st_c32_tiny", "connect4", "small_tower", dict(channels=32, blocks=1), weights="tiny"),
    NetCase("st_1x2_b0", "connect4", "small_tower", _board(1, 2, 2, c=16, blocks=0, **_HEADS16)),

    NetCase("pl_9x9_c32", "connect4", "per_layer", _board(9, 9, 9, c=32, blocks=1)),
    NetCase("pl_c48_6x7", "connect4", "per_layer", dict(channels=48)),
    NetCase("pl_3x3_nofuse", "tictactoe", "per_layer", env=dict(MZ_NO_FUSE="1")),
    NetCase("pl_9x9_wide", "connect4", "per_layer", _board(9, 9, 9, c=32, blocks=1), weights="wide"),
    NetCase("pl_c96_6x7", "connect4", "per_layer", dict(channels=96, blocks=1)),

    NetCase("ss_3x3_a2_c8", "tictactoe", "small_search", _board(3, 3, 2, c=8, blocks=1)),
    NetCase("ss_3x3_a16_c20", "tictactoe", "small_search", _board(3, 3, 16, c=20, blocks=2)),
    NetCase("ss_5x6_a4", "tictactoe", "small_search", _board(5, 6, 4, c=16, blocks=1)),
    NetCase("ss_7x3_a12", "tictactoe", "small_search", _board(7, 3, 12, c=16, blocks=1)),
    NetCase("ss_5x6_tiny", "tictactoe", "small_search", _board(5, 6, 4, c=16, blocks=1), weights="tiny"),

    NetCase("hw_c128_6x7", "connect4", "heads_wide", dict(channels=128, blocks=1)),
    NetCase("hb_c32_6x7", "connect4", "heads_big", dict(channels=32, blocks=1, reduced_channels_value=16,
                                                          resnet_fc_value_layers=[128])),
    NetCase("ds_20x24", "connect4", "downsample", dict(observation_shape=(3, 20, 24), action_space=list(range(4)),
                                                       channels=16, blocks=1, downsample="resnet", **_HEADS16)),
    NetCase("ds_c96_20x24", "connect4", "downsample", dict(observation_shape=(3, 20, 24), action_space=list(range(4)),
                                                           channels=96, blocks=1, downsample="resnet", **_HEADS16)),
    NetCase("ds_33x17", "connect4", "downsample", dict(observation_shape=(3, 33, 17), action_space=list(range(4)),
                                                       channels=16, blocks=1, downsample="resnet", **_HEADS16)),
    NetCase("ds_c8_1x1", "connect4", "downsample", dict(observation_shape=(3, 1, 1), action_space=list(range(4)),
                                                        channels=8, blocks=1, downsample="resnet", **_HEADS16)),
    NetCase("ds_breakout_96x96", "breakout", "downsample"),
    NetCase("ds_atari_96x96", "atari", "downsample", dict(blocks=1), batches=(1, 2, 3)),
    NetCase("ds_atari_96x96_wide", "atari", "downsample", dict(blocks=1), env=dict(MZ_TC_WIDE="3"), batches=(1, 2, 3)),
]

BY_NAME = {c.name: c for c in CASES}

# in-search parity: one case per residual route (the tensor-core case in x3 with one and two graph partitions and in
# fp16; the 6-block tensor-core case, whose gathered dynamics tower is split across launches, with two partitions; the
# nets kept off the tensor cores by their heads, in fp16 and x3) and every FC route
SEARCH_CASES = ["pl_9x9_c32", "pl_c96_6x7", "st_c32_6x7", "ss_5x6_a4", "ss_7x3_a12", "tc_6x7", "tc_6x7_b6", "tc_6x7_s300",
                "tc_6x7_bigheads", "fc_cartpole", "fc_cartpole_s20", "fc_e5_a3", "fc_a40", "ds_breakout_96x96",
                "ds_atari_96x96", "ds_atari_96x96_wide"]


def make_config(case: NetCase):
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module(case.game).MuZeroConfig()
    for k, v in case.over.items():
        setattr(cfg, k, copy.deepcopy(v))
    return cfg


def case_spec(case: NetCase):
    return netspec_from_config(make_config(case))


# ---------------------------------------------------------------------------------------------- small-search planner
def small_search_inputs(spec):
    """Arguments of mz_debug_small_search_plan for a net: the float counts of the tower weights (dynamics stem +
    blocks, prediction blocks), of the heads and of one warp's head scratch, as resnet.cu::small_search_build derives
    them."""
    C, (H, W), A, nb = spec.channels, spec.hidden_hw, spec.action_space, spec.blocks
    r4 = lambda x: (x + 3) & ~3
    dyn = (C + 1) * 9 * C + C + 2 * nb * (C * 9 * C + C)
    pred = 2 * nb * (C * 9 * C + C)
    tower = r4(dyn) + r4(pred)
    heads = 0
    maxw = 32
    for rc, hidden, out in ((spec.reduced_reward, spec.res_fc_reward, spec.full_support),
                            (spec.reduced_value, spec.res_fc_value, spec.full_support),
                            (spec.reduced_policy, spec.res_fc_policy, A)):
        heads = r4(heads) + rc * C + rc
        sizes = [rc * H * W] + list(hidden) + [out]
        for i in range(len(sizes) - 1):
            heads = r4(heads) + ((sizes[i] + 3) // 4) * 4 * sizes[i + 1] + sizes[i + 1]
        maxw = max([maxw, rc * H * W + 4] + [s + 4 for s in sizes[1:]])
    scratch = r4(H * W * (C + 4) + 6 * C + 4 * r4(maxw))
    return dict(H=H, W=W, C=C, A=A, tower=tower, heads=r4(heads), scratch=scratch, cap=C + 1)


# ---------------------------------------------------------------------------------------------- weights
def _towers(spec, w, which=("representation_network.module", "dynamics_network.module")):
    """Per tower: (stem conv key, stem bn prefix, [(conv2 key, bn2 prefix) of every block])."""
    out = []
    for p in which:
        blocks = [(f"{p}.resblocks.{i}.conv2.weight", f"{p}.resblocks.{i}.bn2") for i in range(spec.blocks)]
        out.append((f"{p}.conv.weight", f"{p}.bn", blocks))
    return out


def edge_weights(spec, kind, seed=0, channel=5):
    """``synthetic_weights`` edited into one of the edge cases listed in the module docstring."""
    if kind in ("large", "tiny_bn", "overflow"):
        return stress_weights(spec, seed, {"tiny_bn": "tiny"}.get(kind, kind))
    w = synthetic_weights(spec, seed)
    if kind == "synthetic":
        return w
    f32 = numpy.float32
    c = channel
    if kind in ("const", "tiny"):
        assert spec.kind == RESNET and not spec.downsample
        for stem, bn, blocks in _towers(spec, w):
            # BN shift of channel c = 0: the channel is relu(scale * conv) (and exactly 0 for "const")
            w[f"{bn}.bias"][c] = 0.0
            w[f"{bn}.running_mean"][c] = 0.0
            w[stem][c] = 0.0 if kind == "const" else (w[stem][c] * 3e-7).astype(f32)
            for conv2, bn2 in blocks:
                w[conv2][c] = 0.0
                w[f"{bn2}.bias"][c] = 0.0
                w[f"{bn2}.running_mean"][c] = 0.0
            if kind == "const":        # relu(0 * conv + 0) = 0 everywhere: make it a nonzero constant instead
                w[f"{bn}.bias"][c] = 0.75
        return w
    if kind == "wide":
        assert spec.blocks >= 1
        C = spec.channels
        mags = 10.0 ** numpy.linspace(-8.0, 3.0, C)
        for p in ("representation_network.module", "dynamics_network.module", "prediction_network.module"):
            key = f"{p}.resblocks.{spec.blocks - 1}.conv2.weight"
            rows = w[key].reshape(C, -1)
            rows = rows / numpy.abs(rows).max(1, keepdims=True) * mags[:, None]
            rows[C // 2] = 0.0
            w[key] = rows.reshape(w[key].shape).astype(f32)
        return w
    if kind == "sat":
        for key in ("prediction_network.module.fc_value", "dynamics_network.module.fc"):
            last = max(int(k[len(key) + 1:].split(".")[0]) for k in w if k.startswith(key + ".") and k.endswith(".weight"))
            for leaf in ("weight", "bias"):
                k = f"{key}.{last}.{leaf}"
                w[k] = (w[k] * 40.0).astype(f32)
        return w
    raise ValueError(kind)
