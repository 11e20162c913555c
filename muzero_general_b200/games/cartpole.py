"""CartPole plug-in without gym.

The reference wraps ``gym.make("CartPole-v1")`` (``games/cartpole.py:131-174``); gym 0.21 is a
third-party dependency that is neither vendored in the reference nor installed here, so the
classic cart-pole equations (Barto, Sutton & Anderson 1983; Euler integration, 20 ms step,
episode cap 500, +1 reward per step, termination at |x|>2.4 or |theta|>12 deg) are restated
as a struct-of-arrays numpy environment.  PARITY UNPINNED against gym (absent); it is outside
the hot path (SURVEY.md 8f rank 1) and only provides observations of the right shape and law.
"""
import math

import numpy

from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame, VectorGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "cartpole"
    _OVERRIDES = {}          # the shared defaults ARE the CartPole values


_GRAVITY, _M_CART, _M_POLE, _HALF_LEN, _FORCE, _DT = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
_X_LIMIT = 2.4
_THETA_LIMIT = 12 * 2 * math.pi / 360
_EPISODE_CAP = 500


class CartPoleVector(VectorGame):
    def __init__(self, num_games, seed=None):
        self.num_games = int(num_games)
        self.rs = numpy.random.RandomState(seed)
        self.state = numpy.zeros((self.num_games, 4), dtype=numpy.float64)
        self.steps = numpy.zeros(self.num_games, dtype=numpy.int64)
        self.reset()

    def observations(self):
        return self.state.astype(numpy.float32).reshape(self.num_games, 1, 1, 4)

    def reset(self, which=None):
        if which is None:
            which = numpy.ones(self.num_games, dtype=bool)
        which = numpy.asarray(which)
        n = int(which.sum()) if which.dtype == bool else len(which)
        self.state[which] = self.rs.uniform(-0.05, 0.05, size=(n, 4))
        self.steps[which] = 0
        return self.observations()

    def step(self, actions):
        x, xd, th, thd = self.state.T
        force = numpy.where(numpy.asarray(actions) == 1, _FORCE, -_FORCE)
        cos, sin = numpy.cos(th), numpy.sin(th)
        total = _M_CART + _M_POLE
        pml = _M_POLE * _HALF_LEN
        tmp = (force + pml * thd * thd * sin) / total
        thacc = (_GRAVITY * sin - cos * tmp) / (_HALF_LEN * (4.0 / 3.0 - _M_POLE * cos * cos / total))
        xacc = tmp - pml * thacc * cos / total
        self.state = numpy.stack([x + _DT * xd, xd + _DT * xacc, th + _DT * thd, thd + _DT * thacc], axis=1)
        self.steps += 1
        done = ((numpy.abs(self.state[:, 0]) > _X_LIMIT) | (numpy.abs(self.state[:, 2]) > _THETA_LIMIT)
                | (self.steps >= _EPISODE_CAP))
        return self.observations(), numpy.ones(self.num_games), done

    def legal_mask(self):
        return numpy.ones((self.num_games, 2), dtype=numpy.uint8)


class Game(AbstractGame):
    """Single-game facade with the reference's return shapes (obs (1,1,4), reward 1.0)."""
    DEVICE_ENV = "cartpole"        # the same dynamics exist as a device-resident environment (csrc/selfplay.cu)

    def __init__(self, seed=None):
        self.env = CartPoleVector(1, seed)

    @classmethod
    def vector(cls, num_games, seed=None):
        return CartPoleVector(num_games, seed)

    def step(self, action):
        obs, reward, done = self.env.step(numpy.array([action]))
        return obs[0], float(reward[0]), bool(done[0])

    def legal_actions(self):
        return list(range(2))

    @staticmethod
    def legal_masks(observations):
        """The legal mask of each raw frame [n, *observation_shape] (Reanalyse's hook): every action, as legal_actions."""
        return numpy.ones((len(observations), 2), numpy.uint8)

    def reset(self):
        return self.env.reset()[0]

    def render(self):
        print(self.env.state[0])

    def action_to_string(self, action_number):
        return f"{action_number}. " + ("Push cart to the left", "Push cart to the right")[action_number]
