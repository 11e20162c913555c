"""Network shape description derived from a reference ``MuZeroConfig``.

The reference builds its networks in ``models.py:7-41`` (factory), ``models.py:80-126``
(fully connected) and ``models.py:436-520`` (residual).  This module derives, from the
config attribute bag alone, everything the CUDA side needs to know:

* ``NetSpec`` - the POD description handed to the C-ABI (``include/mzb200.h``),
* ``weights_spec`` - the ordered ``(state_dict key, shape)`` list of the reference's
  ``get_weights()`` (``models.py:69-70``), including the ``.module.`` infix that
  ``torch.nn.DataParallel`` adds (``models.py:98-126,486-520``) and the unused
  ``conv``/``bn`` the reference still registers when ``downsample`` is set
  (``models.py:330-337``).

Nothing here touches the GPU.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Tuple

FC = 0
RESNET = 1


@dataclass
class NetSpec:
    kind: int                       # FC or RESNET
    obs_shape: Tuple[int, int, int]  # (C, H, W) of ONE raw observation
    stacked: int                    # config.stacked_observations
    in_channels: int                # C*(s+1)+s   (self_play.py:513-550, models.py:100-104)
    action_space: int
    support_size: int
    # FC
    encoding: int = 0
    fc_representation: List[int] = field(default_factory=list)
    fc_dynamics: List[int] = field(default_factory=list)
    fc_reward: List[int] = field(default_factory=list)
    fc_value: List[int] = field(default_factory=list)
    fc_policy: List[int] = field(default_factory=list)
    # ResNet
    blocks: int = 0
    channels: int = 0
    reduced_reward: int = 0
    reduced_value: int = 0
    reduced_policy: int = 0
    res_fc_reward: List[int] = field(default_factory=list)
    res_fc_value: List[int] = field(default_factory=list)
    res_fc_policy: List[int] = field(default_factory=list)
    downsample: int = 0             # 0 none, 1 "resnet" (models.py:233-275), 2 "CNN" (models.py:278-297)

    @property
    def full_support(self) -> int:
        return 2 * self.support_size + 1

    @property
    def obs_elems(self) -> int:
        return self.in_channels * self.obs_shape[1] * self.obs_shape[2]

    @property
    def hidden_hw(self) -> Tuple[int, int]:
        """Spatial size of the hidden state (models.py:456-484)."""
        if self.kind == FC:
            return (1, 1)
        if self.downsample:
            return (math.ceil(self.obs_shape[1] / 16), math.ceil(self.obs_shape[2] / 16))
        return (self.obs_shape[1], self.obs_shape[2])

    @property
    def hidden_elems(self) -> int:
        if self.kind == FC:
            return self.encoding
        h, w = self.hidden_hw
        return self.channels * h * w


def netspec_from_config(config) -> NetSpec:
    """Read exactly the attributes ``models.MuZeroNetwork.__new__`` reads (models.py:7-41)."""
    c, h, w = config.observation_shape
    s = config.stacked_observations
    common = dict(
        obs_shape=(int(c), int(h), int(w)),
        stacked=int(s),
        in_channels=int(c) * (s + 1) + s,
        action_space=len(config.action_space),
        support_size=int(config.support_size),
    )
    if config.network == "fullyconnected":
        return NetSpec(
            kind=FC,
            encoding=int(config.encoding_size),
            fc_representation=list(config.fc_representation_layers),
            fc_dynamics=list(config.fc_dynamics_layers),
            fc_reward=list(config.fc_reward_layers),
            fc_value=list(config.fc_value_layers),
            fc_policy=list(config.fc_policy_layers),
            **common,
        )
    if config.network == "resnet":
        ds = config.downsample
        if ds not in (False, None, 0, "resnet", "CNN"):
            raise NotImplementedError('downsample should be "resnet" or "CNN".')
        return NetSpec(
            kind=RESNET,
            blocks=int(config.blocks),
            channels=int(config.channels),
            reduced_reward=int(config.reduced_channels_reward),
            reduced_value=int(config.reduced_channels_value),
            reduced_policy=int(config.reduced_channels_policy),
            res_fc_reward=list(config.resnet_fc_reward_layers),
            res_fc_value=list(config.resnet_fc_value_layers),
            res_fc_policy=list(config.resnet_fc_policy_layers),
            downsample={False: 0, None: 0, 0: 0, "resnet": 1, "CNN": 2}[ds],
            **common,
        )
    raise NotImplementedError('The network parameter should be "fullyconnected" or "resnet".')


# --------------------------------------------------------------------------------------
# state_dict layout
# --------------------------------------------------------------------------------------
def _mlp_keys(prefix: str, sizes: List[int]):
    """``mlp`` (models.py:630-642): Linear at Sequential index 0, 2, 4, ..."""
    out = []
    for i in range(len(sizes) - 1):
        out.append((f"{prefix}.{2 * i}.weight", (sizes[i + 1], sizes[i])))
        out.append((f"{prefix}.{2 * i}.bias", (sizes[i + 1],)))
    return out


def _bn_keys(prefix: str, ch: int):
    return [
        (f"{prefix}.weight", (ch,)),
        (f"{prefix}.bias", (ch,)),
        (f"{prefix}.running_mean", (ch,)),
        (f"{prefix}.running_var", (ch,)),
        (f"{prefix}.num_batches_tracked", ()),
    ]


def _resblock_keys(prefix: str, ch: int):
    out = [(f"{prefix}.conv1.weight", (ch, ch, 3, 3))]
    out += _bn_keys(f"{prefix}.bn1", ch)
    out += [(f"{prefix}.conv2.weight", (ch, ch, 3, 3))]
    out += _bn_keys(f"{prefix}.bn2", ch)
    return out


def weights_spec(spec: NetSpec):
    """Ordered (key, shape) list equal to the reference ``state_dict()`` for this config."""
    A, F = spec.action_space, spec.full_support
    keys = []
    if spec.kind == FC:
        E = spec.encoding
        keys += _mlp_keys("representation_network.module", [spec.obs_elems] + spec.fc_representation + [E])
        keys += _mlp_keys("dynamics_encoded_state_network.module", [E + A] + spec.fc_dynamics + [E])
        keys += _mlp_keys("dynamics_reward_network.module", [E] + spec.fc_reward + [F])
        keys += _mlp_keys("prediction_policy_network.module", [E] + spec.fc_policy + [A])
        keys += _mlp_keys("prediction_value_network.module", [E] + spec.fc_value + [F])
        return keys

    C = spec.channels
    hh, hw = spec.hidden_hw
    rp = "representation_network.module"
    if spec.downsample == 1:
        dp = f"{rp}.downsample_net"
        keys += [(f"{dp}.conv1.weight", (C // 2, spec.in_channels, 3, 3))]
        for i in range(2):
            keys += _resblock_keys(f"{dp}.resblocks1.{i}", C // 2)
        keys += [(f"{dp}.conv2.weight", (C, C // 2, 3, 3))]
        for i in range(3):
            keys += _resblock_keys(f"{dp}.resblocks2.{i}", C)
        for i in range(3):
            keys += _resblock_keys(f"{dp}.resblocks3.{i}", C)
    elif spec.downsample == 2:
        # DownsampleCNN (models.py:278-297): conv k x k (k = 2 * ceil(H / 16)) to (in + C) // 2 channels, conv 5 x 5 to C
        mid, k = (spec.in_channels + C) // 2, 2 * hh
        dp = f"{rp}.downsample_net.features"
        keys += [(f"{dp}.0.weight", (mid, spec.in_channels, k, k)), (f"{dp}.0.bias", (mid,)),
                 (f"{dp}.3.weight", (C, mid, 5, 5)), (f"{dp}.3.bias", (C,))]
    keys += [(f"{rp}.conv.weight", (C, spec.in_channels, 3, 3))]
    keys += _bn_keys(f"{rp}.bn", C)
    for i in range(spec.blocks):
        keys += _resblock_keys(f"{rp}.resblocks.{i}", C)

    dp = "dynamics_network.module"
    keys += [(f"{dp}.conv.weight", (C, C + 1, 3, 3))]
    keys += _bn_keys(f"{dp}.bn", C)
    for i in range(spec.blocks):
        keys += _resblock_keys(f"{dp}.resblocks.{i}", C)
    keys += [(f"{dp}.conv1x1_reward.weight", (spec.reduced_reward, C, 1, 1)),
             (f"{dp}.conv1x1_reward.bias", (spec.reduced_reward,))]
    keys += _mlp_keys(f"{dp}.fc", [spec.reduced_reward * hh * hw] + spec.res_fc_reward + [F])

    pp = "prediction_network.module"
    for i in range(spec.blocks):
        keys += _resblock_keys(f"{pp}.resblocks.{i}", C)
    keys += [(f"{pp}.conv1x1_value.weight", (spec.reduced_value, C, 1, 1)),
             (f"{pp}.conv1x1_value.bias", (spec.reduced_value,)),
             (f"{pp}.conv1x1_policy.weight", (spec.reduced_policy, C, 1, 1)),
             (f"{pp}.conv1x1_policy.bias", (spec.reduced_policy,))]
    keys += _mlp_keys(f"{pp}.fc_value", [spec.reduced_value * hh * hw] + spec.res_fc_value + [F])
    keys += _mlp_keys(f"{pp}.fc_policy", [spec.reduced_policy * hh * hw] + spec.res_fc_policy + [A])
    return keys


def synthetic_weights(spec: NetSpec, seed: int = 0):
    """Deterministic, reference-independent weights for a config (numpy legacy stream).

    Used by the golden generator, the tests and bench.py: the reference's own
    ``torch.manual_seed(0)`` initialisation depends on its module construction order and
    cannot be reproduced without importing it, whereas ``numpy.random.RandomState`` streams
    are version-stable.  BatchNorm statistics are deliberately non-trivial so BN folding is
    actually exercised.  Returns ``{key: numpy array}`` in ``weights_spec`` order.
    """
    import numpy

    rs = numpy.random.RandomState(seed)
    out = {}
    for key, shape in weights_spec(spec):
        leaf = key.rsplit(".", 1)[1]
        if leaf == "num_batches_tracked":
            out[key] = numpy.array(7, dtype=numpy.int64)
        elif leaf == "running_var":
            out[key] = rs.uniform(0.5, 1.5, size=shape).astype(numpy.float32)
        elif leaf == "running_mean":
            out[key] = (0.1 * rs.standard_normal(size=shape)).astype(numpy.float32)
        elif leaf == "weight" and len(shape) == 1:      # BN gamma
            out[key] = rs.uniform(0.8, 1.2, size=shape).astype(numpy.float32)
        elif leaf == "bias":
            out[key] = (0.1 * rs.standard_normal(size=shape)).astype(numpy.float32)
        else:                                           # conv / linear weight
            fan_in = int(numpy.prod(shape[1:]))
            out[key] = (rs.standard_normal(size=shape) / math.sqrt(fan_in)).astype(numpy.float32)
    return out


def stress_weights(spec: NetSpec, seed: int = 0, mode: str = "large"):
    """``synthetic_weights`` with the BatchNorm affine terms of the residual towers rescaled so that the tower
    activations leave the comfortable O(1) range (the range guard of the tensor-core towers is tested with these):

    * ``"large"``     every tower BN gamma x4: activations grow ~16x per block, up to ~1e3..1e4 (inside fp16 range)
    * ``"overflow"``  every tower BN gamma x12: activations exceed 65504, the largest finite fp16
    * ``"tiny"``      first BN of every block x1e-5 (gamma and beta), second BN gamma x1e5, mean x1e-5: the intermediate
                      activation of a block is ~1e-5 (below the smallest normal fp16) while the block output stays O(1)
    """
    import numpy

    w = synthetic_weights(spec, seed)
    if spec.kind != RESNET:
        raise ValueError("stress_weights is for residual networks")
    for key in list(w):
        parts = key.split(".")
        leaf, bn = parts[-1], parts[-2]
        if not bn.startswith("bn") or "downsample_net" in key:
            continue
        if mode in ("large", "overflow"):
            if leaf == "weight":
                w[key] = (w[key] * (4.0 if mode == "large" else 12.0)).astype(numpy.float32)
        elif mode == "tiny":
            if bn == "bn1" and leaf in ("weight", "bias"):
                w[key] = (w[key] * 1e-5).astype(numpy.float32)
            elif bn == "bn2" and leaf == "weight":
                w[key] = (w[key] * 1e5).astype(numpy.float32)
            elif bn == "bn2" and leaf == "running_mean":
                w[key] = (w[key] * 1e-5).astype(numpy.float32)
        else:
            raise ValueError(f"unknown stress mode {mode!r}")
    return w
