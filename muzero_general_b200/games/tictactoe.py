"""TicTacToe plug-in (config values and rules of the reference's ``games/tictactoe.py``)."""
import numpy

from ._boards import BoardGame, BoardVector
from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "tictactoe"
    _OVERRIDES = dict(
        observation_shape=(3, 3, 3), action_space=list(range(9)), players=list(range(2)),
        opponent="expert", max_moves=9, num_simulations=25, discount=1,
        root_dirichlet_alpha=0.1,
        network="resnet", blocks=1, channels=16,
        reduced_channels_reward=16, reduced_channels_value=16, reduced_channels_policy=16,
        resnet_fc_reward_layers=[8], resnet_fc_value_layers=[8], resnet_fc_policy_layers=[8],
        encoding_size=32, fc_value_layers=[], fc_policy_layers=[],
        training_steps=1000000, batch_size=64, value_loss_weight=0.25, lr_init=0.003,
        lr_decay_rate=1, lr_decay_steps=10000, replay_buffer_size=3000, num_unroll_steps=20,
        td_steps=20, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((None, 1),)


class TicTacToeVector(BoardVector):
    H = W = K = 3
    OBS_DTYPE = numpy.int32
    REWARD_SCALE = 20          # games/tictactoe.py:144

    @staticmethod
    def expert_windows(board):
        """Scan order of games/tictactoe.py:313-347: row i then column i for i = 0..2, diagonal, anti-diagonal."""
        class Any:
            def __call__(self, y, x): return True
            @staticmethod
            def action(y, x): return y * 3 + x
        ok = Any()
        out = []
        for i in range(3):
            out.append(([(i, 0), (i, 1), (i, 2)], 2, ok, None))
            out.append(([(0, i), (1, i), (2, i)], 2, ok, None))
        out.append(([(0, 0), (1, 1), (2, 2)], 2, ok, None))
        out.append(([(0, 2), (1, 1), (2, 0)], 2, ok, None))      # numpy.fliplr(board).diagonal(): index j <-> (j, 2 - j)
        return out


class Game(BoardGame, AbstractGame):
    DEVICE_ENV = "tictactoe"        # csrc/selfplay.cu restates these rules on the device
    VECTOR = TicTacToeVector

    def action_to_string(self, action_number):
        return f"Play row {action_number // 3 + 1}, column {action_number % 3 + 1}"

    def _expert_windows(self, board):
        return TicTacToeVector.expert_windows(board)

    def human_to_action(self):
        while True:
            try:
                row = int(input(f"Enter the row (1, 2 or 3) to play for the player {self.to_play()}: "))
                col = int(input(f"Enter the column (1, 2 or 3) to play for the player {self.to_play()}: "))
                choice = (row - 1) * 3 + (col - 1)
                if choice in self.legal_actions() and 1 <= row <= 3 and 1 <= col <= 3:
                    return choice
            except ValueError:
                pass
            print("Wrong input, try again")
