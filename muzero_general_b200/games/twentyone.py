"""Twenty-One plug-in (config values and rules of the reference's ``games/twentyone.py``): one player against a
dealer who draws to 17; an ace counts 1.  The rules take their cards from a pluggable source - the reference's
``numpy.random.RandomState(seed).randint(1, 13)`` by default - so the same code replays any card stream."""
import numpy

from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame, VectorGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "twentyone"
    _OVERRIDES = dict(
        observation_shape=(3, 3, 3), num_workers=4, max_moves=21, num_simulations=21, discount=1,
        network="resnet", blocks=2, channels=32,
        reduced_channels_reward=32, reduced_channels_value=32, reduced_channels_policy=32,
        resnet_fc_reward_layers=[16], resnet_fc_value_layers=[16], resnet_fc_policy_layers=[16],
        encoding_size=32, fc_representation_layers=[16],
        training_steps=15000, batch_size=64, value_loss_weight=0.25, optimizer="SGD", lr_init=0.03,
        lr_decay_rate=0.75, lr_decay_steps=150000, replay_buffer_size=10000, num_unroll_steps=20, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((500e3, 1.0), (750e3, 0.5), (None, 0.25))
    _TEMPERATURE_ABSOLUTE = True


def numpy_cards(seed):
    """``TwentyOne.deal_card_value`` (games/twentyone.py:288-294): a card of ``randint(1, 13)``, faces counting 10."""
    rs = numpy.random.RandomState(seed)

    def deal():
        return min(int(rs.randint(1, 13)), 10)
    return deal


class TwentyOneVector(VectorGame):
    """``num_games`` tables (games/twentyone.py:228-303).  ``cards[g]`` is game g's card source, a callable returning
    the next card's value; by default ``numpy_cards(seed + g)``.  ``reset`` deals the player's card, then the
    dealer's; a hit deals one card; when the game ends the dealer draws while at 16 or less, unless the player went
    bust.  Rewards are ``get_reward`` times ``REWARD_SCALE`` (``Game.step``'s x10)."""
    OBS_DTYPE = numpy.float64      # the reference's [float32 plane, float32 plane, int64 plane] as one array
    REWARD_SCALE = 10

    def __init__(self, num_games, seed=None, cards=None):
        self.num_games = int(num_games)
        if cards is None:
            cards = [numpy_cards(None if seed is None else seed + g) for g in range(self.num_games)]
        self.cards = list(cards)
        self.player = numpy.zeros(self.num_games, dtype=numpy.int64)
        self.dealer = numpy.zeros(self.num_games, dtype=numpy.int64)

    def reset(self, which=None):
        idx = range(self.num_games) if which is None else numpy.arange(self.num_games)[numpy.asarray(which)]
        for g in idx:
            self.player[g] = self.cards[g]()
            self.dealer[g] = self.cards[g]()
        return self.observations()

    def observations(self):
        obs = numpy.zeros((self.num_games, 3, 3, 3), dtype=self.OBS_DTYPE)
        obs[:, 0] = self.player[:, None, None]
        obs[:, 1] = self.dealer[:, None, None]
        return obs

    def legal_mask(self):
        return numpy.ones((self.num_games, 2), dtype=numpy.uint8)

    def step(self, actions):
        rewards = numpy.zeros(self.num_games, dtype=numpy.int64)
        dones = numpy.zeros(self.num_games, dtype=bool)
        for g, a in enumerate(numpy.asarray(actions).tolist()):
            if a == 0:
                self.player[g] += self.cards[g]()
            p = int(self.player[g])
            done = p > 21 or a == 1 or p == 21
            if done:
                if p <= 21:
                    while self.dealer[g] <= 16:
                        self.dealer[g] += self.cards[g]()
                d = int(self.dealer[g])
                if p <= 21 and (d < p or d > 21):
                    rewards[g] = 1
                elif p > 21 or p != d:
                    rewards[g] = -1
            dones[g] = done
        return self.observations(), rewards * self.REWARD_SCALE, dones


class Game(AbstractGame):
    DEVICE_ENV = "twentyone"        # csrc/selfplay.cu restates these rules on the device
    VECTOR = TwentyOneVector

    def __init__(self, seed=None):
        self.env = TwentyOneVector(1, seed)
        self.env.reset()            # TwentyOne.__init__ deals two cards before reset deals the game's own

    @classmethod
    def vector(cls, num_games, seed=None):
        env = TwentyOneVector(num_games, seed)
        env.reset()                 # as Game(seed + g) does
        return env

    def step(self, action):
        obs, reward, done = self.env.step(numpy.array([action]))
        return obs[0], int(reward[0]), bool(done[0])

    def legal_actions(self):
        return [0, 1]

    @staticmethod
    def legal_masks(observations):
        """The legal mask of each raw frame [n, *observation_shape] (Reanalyse's hook): every action, as legal_actions."""
        return numpy.ones((len(observations), 2), numpy.uint8)

    def reset(self):
        return self.env.reset()[0]

    def render(self):
        print("Dealer hand: " + str(int(self.env.dealer[0])))
        print("Player hand: " + str(int(self.env.player[0])))

    def human_to_action(self):
        choice = input(f"Enter the action (0) Hit, or (1) Stand for the player {self.to_play()}: ")
        while choice not in [str(action) for action in self.legal_actions()]:
            choice = input("Enter either (0) Hit or (1) Stand : ")
        return int(choice)

    def action_to_string(self, action_number):
        return f"{action_number}. " + ("Hit", "Stand")[action_number]
