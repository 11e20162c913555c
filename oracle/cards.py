"""ORACLE (test infrastructure). Twenty-One's card stream on the device, restated on the CPU.

``twentyone_card`` (``muzero_general_b200/csrc/selfplay.cu``) draws card k of a game from the Philox4x32-10 stream
tag 0x7169E006 through ``philox_uniform53``, restated as ``oracle.philox.uniform53``; the bit recipe is checked in
``tests/test_device_games_cpu.py``.
"""
from oracle.philox import uniform53

TAG_CARD = 0x7169E006


def card(seed, game, k):
    """Twenty-One's draw k of a game: u = ``uniform53`` at counter (game_lo, k, 0, game_hi) under TAG_CARD,
    card = 1 + floor(12 u) like ``randint(1, 13)``, worth min(card, 10).  Draw 0 is the player's first card, draw 1
    the dealer's, then every hit and the dealer's draws in the reference's order."""
    return min(1 + int(12.0 * uniform53(seed, game, k, 0, TAG_CARD)), 10)
