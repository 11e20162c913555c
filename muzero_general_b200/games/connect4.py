"""Connect4 plug-in (config values and rules of the reference's ``games/connect4.py``)."""
import numpy

from ._boards import BoardGame, BoardVector
from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "connect4"
    _OVERRIDES = dict(
        observation_shape=(3, 6, 7), action_space=list(range(7)), players=list(range(2)),
        opponent="expert", max_moves=42, num_simulations=200, discount=1,
        root_dirichlet_alpha=0.3,
        network="resnet", blocks=3, channels=64,
        reduced_channels_reward=2, reduced_channels_value=2, reduced_channels_policy=4,
        resnet_fc_reward_layers=[64], resnet_fc_value_layers=[64], resnet_fc_policy_layers=[64],
        encoding_size=32, fc_dynamics_layers=[64], fc_reward_layers=[64],
        fc_value_layers=[], fc_policy_layers=[],
        training_steps=100000, batch_size=64, value_loss_weight=0.25, lr_init=0.005,
        lr_decay_rate=1, lr_decay_steps=10000, replay_buffer_size=10000, num_unroll_steps=42,
        td_steps=42, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((None, 1),)


class Connect4Vector(BoardVector):
    H, W, K = 6, 7, 4
    GRAVITY = True
    OBS_DTYPE = numpy.float64
    REWARD_SCALE = 10          # games/connect4.py:144

    @staticmethod
    def expert_windows(board):
        """Scan order of games/connect4.py:310-346: 4x4 sub-boards (k = 0..2 rows up, l = 0..3 columns right); inside
        one: for i = 0..3 the i-th row then the i-th column, then the diagonal, then the anti-diagonal.  A gap counts
        only when it is the next free cell of its column; the vertical check plays its column unconditionally."""
        heights = [int(numpy.count_nonzero(board[:, x])) for x in range(7)]

        class NextFree:
            def __call__(self, y, x): return heights[x] == y
            @staticmethod
            def action(y, x): return x
        ok = NextFree()
        out = []
        for k in range(3):
            for l in range(4):
                for i in range(4):
                    out.append(([(k + i, l + j) for j in range(4)], 3, ok, None))
                    out.append(([(k + j, l + i) for j in range(4)], 3, ok, l + i))
                out.append(([(k + j, l + j) for j in range(4)], 3, ok, None))
                out.append(([(k + j, l + 3 - j) for j in range(4)], 3, ok, None))
        return out


class Game(BoardGame, AbstractGame):
    DEVICE_ENV = "connect4"        # csrc/selfplay.cu restates these rules on the device
    VECTOR = Connect4Vector

    def action_to_string(self, action_number):
        return f"Play column {action_number + 1}"

    def human_to_action(self):
        choice = input(f"Enter the column to play for the player {self.to_play()}: ")
        while choice not in [str(action) for action in self.legal_actions()]:
            choice = input("Enter another column : ")
        return int(choice)

    def _expert_windows(self, board):
        return Connect4Vector.expert_windows(board)
