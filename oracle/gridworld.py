"""ORACLE (test infrastructure). Gridworld's placement on the device, restated on the CPU.

``gridworld_reset`` (``muzero_general_b200/csrc/selfplay.cu``) places the agent of a game from two draws of the
Philox4x32-10 stream tag 0x7169E007 through ``philox_uniform53``, restated as ``oracle.philox.uniform53``; the bit
recipe is checked in ``tests/test_gridworld_cpu.py``.
"""
from oracle.philox import uniform53

TAG_PLACE = 0x7169E007


def placement(seed, game):
    """Gridworld's placement of a game: u_k = ``uniform53`` at counter (game_lo, k, 0, game_hi) under TAG_PLACE for
    draws k = 0 and 1.  The cell is the floor(15 u_0)-th free cell in the order (1, 1), (2, 1), (3, 1), (4, 1), (1, 2),
    ..., (3, 4), that is x = 1 + i % 4, y = 1 + i // 4 (the goal (4, 4) would be i = 15); the direction is
    floor(4 u_1).  Returns (x, y, dir)."""
    i = int(15.0 * uniform53(seed, game, 0, 0, TAG_PLACE))
    return 1 + i % 4, 1 + i // 4, int(4.0 * uniform53(seed, game, 1, 0, TAG_PLACE))
