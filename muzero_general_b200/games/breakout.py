"""Breakout-shaped plug-in with synthetic frames.

The reference wraps ALE ``Breakout-v4`` + ``cv2.resize`` (``games/breakout.py:136-199``); ALE is
not available here, so this stand-in keeps the reference's CONFIG (network, observation
shape (3,96,96) float32 in [0,1), 4 always-legal actions) and produces frames from
``numpy.random.RandomState(seed)`` with a fixed episode length (SURVEY.md 8d).  It exists to
feed the representation network of BASELINE config 5 with inputs of the right shape.
"""
import numpy

from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame, VectorGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "breakout"
    _OVERRIDES = dict(
        observation_shape=(3, 96, 96), action_space=list(range(4)), players=list(range(1)),
        max_moves=2500, num_simulations=30, discount=0.997,
        network="resnet", downsample="resnet", blocks=2, channels=16,
        reduced_channels_reward=4, reduced_channels_value=4, reduced_channels_policy=4,
        resnet_fc_reward_layers=[16], resnet_fc_value_layers=[16], resnet_fc_policy_layers=[16],
        encoding_size=10, fc_value_layers=[], fc_policy_layers=[],
        training_steps=int(1000e3), batch_size=16, checkpoint_interval=500, value_loss_weight=0.25,
        lr_init=0.005, lr_decay_rate=1, lr_decay_steps=350e3,
        replay_buffer_size=int(1e6), num_unroll_steps=5, td_steps=10, PER_alpha=1,
        use_last_model_value=False, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((500e3, 1.0), (750e3, 0.5), (None, 0.25))
    _TEMPERATURE_ABSOLUTE = True


class SyntheticFramesVector(VectorGame):
    EPISODE = 64

    def __init__(self, num_games, seed=None):
        self.num_games = int(num_games)
        self.rs = numpy.random.RandomState(seed)
        self.t = numpy.zeros(self.num_games, dtype=numpy.int64)
        self._obs = None
        self.reset()

    def observations(self):
        return self._obs

    def reset(self, which=None):
        if which is None or self._obs is None:
            self._obs = self.rs.random_sample((self.num_games, 3, 96, 96)).astype(numpy.float32)
            self.t[:] = 0
        else:
            n = int(numpy.asarray(which).sum())
            self._obs[which] = self.rs.random_sample((n, 3, 96, 96)).astype(numpy.float32)
            self.t[which] = 0
        return self._obs

    def step(self, actions):
        self._obs = self.rs.random_sample((self.num_games, 3, 96, 96)).astype(numpy.float32)
        self.t += 1
        reward = (numpy.asarray(actions) == (self.t % 4)).astype(numpy.float64)
        return self._obs, reward, self.t >= self.EPISODE

    def legal_mask(self):
        return numpy.ones((self.num_games, 4), dtype=numpy.uint8)


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
