"""Gomoku plug-in (config values and rules of the reference's ``games/gomoku.py``): 11 x 11 board, five in a row,
121 actions - the wide-action-space case of the tree kernels (``csrc/tree_wide.cu``: four actions per lane)."""
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


class GomokuVector(BoardVector):
    H = W = 11
    K = 5
    OBS_DTYPE = numpy.float64
    REWARD_SCALE = 1
    REWARD_WHEN_FULL = True


class Game(BoardGame, AbstractGame):
    DEVICE_ENV = "gomoku"           # csrc/selfplay.cu restates these rules on the device
    VECTOR = GomokuVector

    def action_to_string(self, action_number):
        return chr(action_number // 11 + 65) + chr(action_number % 11 + 65)
