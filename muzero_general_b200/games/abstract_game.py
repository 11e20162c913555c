"""Game plug-in surface kept from the reference (``games/abstract_game.py:4-105``).

Same method names, argument meaning and return conventions, so a reference ``Game`` class
works here unchanged and vice versa.  OPTIONAL additions, all discovered with
``getattr`` so stock plug-ins keep working:

* ``Game.vector(num_games, seed)`` - a classmethod returning a ``VectorGame`` that steps
  ``num_games`` independent copies at once (struct-of-arrays, numpy).  The batched
  self-play loop uses it when present and falls back to ``num_games`` ordinary ``Game``
  objects otherwise.
* ``Game.legal_masks(observations)`` - uint8 ``[n, |A|]``, the legal mask of each raw frame
  ``[n, *observation_shape]``; Reanalyse with ``config.reanalyse_search`` needs it, because a
  ``GameHistory`` stores no legal actions.
"""
from abc import ABC, abstractmethod


class AbstractGame(ABC):
    @abstractmethod
    def __init__(self, seed=None):
        ...

    @abstractmethod
    def step(self, action):
        """Apply ``action``; returns ``(observation[C,H,W], reward, done)``."""

    def to_play(self):
        """Current player, an element of ``config.players``."""
        return 0

    @abstractmethod
    def legal_actions(self):
        """List of ints, a subset of ``config.action_space``."""

    @abstractmethod
    def reset(self):
        """Start a new game; returns the first observation."""

    def close(self):
        pass

    @abstractmethod
    def render(self):
        ...

    def human_to_action(self):
        choice = input(f"Enter the action to play for the player {self.to_play()}: ")
        while int(choice) not in self.legal_actions():
            choice = input("Illegal action. Enter another action : ")
        return int(choice)

    def expert_agent(self):
        raise NotImplementedError

    def action_to_string(self, action_number):
        return str(action_number)


class VectorGame(ABC):
    """``num_games`` independent copies of one game, stepped together (host side, numpy)."""

    num_games: int

    @abstractmethod
    def reset(self, which=None):
        """Reset all games (or the boolean/int-indexed subset ``which``); returns all observations."""

    @abstractmethod
    def step(self, actions):
        """actions: int array [num_games] -> (obs [n,C,H,W], reward [n], done [n] bool)."""

    @abstractmethod
    def legal_mask(self):
        """uint8 [num_games, |A|]"""

    def to_play(self):
        import numpy
        return numpy.zeros(self.num_games, dtype=numpy.int32)

    def observations(self):
        raise NotImplementedError
