"""Gomoku plug-in (config values and rules of the reference's ``games/gomoku.py``): five in a row on a
``board_size`` x ``board_size`` board, 11 by default like the reference's ``Gomoku.board_size`` - the wide-action-space
case of the tree kernels (``csrc/tree_wide.cu``: four actions per lane up to 128 actions, eight up to 256).  The device
loop plays sides 5 to 16 and reads the side from the action space, so ``MuZeroConfig(board_size=15)`` is all it needs;
the host loop builds its environments from the ``Game`` class, so it takes ``Game.sized(15)``."""
import numpy

from ._boards import BoardGame, BoardVector
from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "gomoku"
    _OVERRIDES = dict(
        observation_shape=(3, 11, 11), action_space=list(range(11 * 11)), players=list(range(2)),
        opponent="random", num_workers=2, max_moves=121, num_simulations=400, discount=1,
        root_dirichlet_alpha=0.3,
        network="resnet", blocks=6, channels=128,
        reduced_channels_reward=2, reduced_channels_value=2, reduced_channels_policy=4,
        resnet_fc_reward_layers=[64], resnet_fc_value_layers=[64], resnet_fc_policy_layers=[64],
        encoding_size=32, fc_dynamics_layers=[64], fc_reward_layers=[64],
        fc_value_layers=[], fc_policy_layers=[],
        training_steps=10000, batch_size=512, checkpoint_interval=50, lr_init=0.002,
        lr_decay_rate=0.9, lr_decay_steps=10000, replay_buffer_size=10000, num_unroll_steps=121,
        td_steps=121, use_last_model_value=False, ratio=1,
    )

    def __init__(self, board_size=11):
        super().__init__()
        self.board_size = int(board_size)
        self.observation_shape = (3, self.board_size, self.board_size)
        self.action_space = list(range(self.board_size * self.board_size))


class GomokuVector(BoardVector):
    H = W = 11
    K = 5
    OBS_DTYPE = numpy.float64
    REWARD_SCALE = 1
    REWARD_WHEN_FULL = True

    def __init__(self, num_games, seed=None, board_size=11):
        self.H = self.W = int(board_size)
        super().__init__(num_games, seed)


class Game(BoardGame, AbstractGame):
    DEVICE_ENV = "gomoku"           # csrc/selfplay.cu restates these rules on the device
    VECTOR = GomokuVector
    BOARD_SIZE = 11                 # the side when none is given (the reference's Gomoku.board_size)

    def __init__(self, seed=None, board_size=None):
        self.env = self.VECTOR(1, seed, board_size or self.BOARD_SIZE)

    @classmethod
    def vector(cls, num_games, seed=None, board_size=None):
        return cls.VECTOR(num_games, seed, board_size or cls.BOARD_SIZE)

    @classmethod
    def sized(cls, board_size):
        """The ``Game`` class of another board side, for callers that build games as ``Game(seed)``."""
        return type(cls.__name__, (cls,), {"BOARD_SIZE": int(board_size)})

    def action_to_string(self, action_number):
        return chr(action_number // self.env.W + 65) + chr(action_number % self.env.W + 65)
