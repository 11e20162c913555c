"""Atari-shaped plug-in with synthetic frames: the reference's LARGE configuration (``games/atari.py:17-117``).

32 stacked observations (3*(32+1)+32 = 131 input planes of 96x96), a 16-block / 256-channel residual network behind the
DownSample stem, 256-channel heads with two hidden layers and a support of 601 bins.  ALE is not available here (SURVEY.md
8c), so - like ``games/breakout.py`` - the environment is a stand-in producing frames from ``numpy.random.RandomState``;
the CONFIG is the reference's, which is what exercises the stacked-observation path of ``GameHistory`` /
``BatchedSelfPlay`` and the large-network route of the library (row-banded convolutions, generic heads: resnet.cu).
"""
from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame
from .breakout import SyntheticFramesVector

import numpy


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "atari"
    _OVERRIDES = dict(
        observation_shape=(3, 96, 96), action_space=list(range(4)), players=list(range(1)),
        stacked_observations=32, num_workers=350, max_moves=27000, num_simulations=50, discount=0.997,
        network="resnet", support_size=300, downsample="resnet", blocks=16, channels=256,
        reduced_channels_reward=256, reduced_channels_value=256, reduced_channels_policy=256,
        resnet_fc_reward_layers=[256, 256], resnet_fc_value_layers=[256, 256], resnet_fc_policy_layers=[256, 256],
        encoding_size=10, fc_value_layers=[], fc_policy_layers=[],
        training_steps=int(1000e3), batch_size=1024, checkpoint_interval=int(1e3), value_loss_weight=0.25,
        optimizer="SGD", lr_init=0.05, lr_decay_rate=0.1, lr_decay_steps=350e3,
        replay_buffer_size=int(1e6), num_unroll_steps=5, td_steps=10, PER_alpha=1, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((500e3, 1.0), (750e3, 0.5), (None, 0.25))
    _TEMPERATURE_ABSOLUTE = True


class Game(AbstractGame):
    def __init__(self, seed=None):
        self.env = SyntheticFramesVector(1, seed)

    @classmethod
    def vector(cls, num_games, seed=None):
        return SyntheticFramesVector(num_games, seed)

    def step(self, action):
        obs, reward, done = self.env.step(numpy.array([action]))
        return obs[0], float(reward[0]), bool(done[0])

    def legal_actions(self):
        return list(range(4))

    @staticmethod
    def legal_masks(observations):
        """The legal mask of each raw frame [n, *observation_shape] (Reanalyse's hook): every action, as legal_actions."""
        return numpy.ones((len(observations), 4), numpy.uint8)

    def reset(self):
        return self.env.reset()[0]

    def render(self):
        print("synthetic frame", self.env.t[0])
