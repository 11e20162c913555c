"""CTA size of the fused FC search (csrc/fc_search.cu::fc_search_plan, host arithmetic only).

The kernel is latency-bound, so a launch lasts about one game's chain of simulations per pass of its persistent loop:
the planner takes the CTA size whose resident CTAs hold the batch in the fewest passes, then the smallest CTA.  Device
figures are the H100's: 132 SMs, 233472 B of shared memory per SM, 1024 B of it reserved per CTA, 232448 B at most per
CTA; the kernel runs at 128 registers per thread."""
import ctypes as C

import pytest

H100 = dict(sms=132, smem_per_sm=233472, reserve=1024, cap=232448, regs=128)
# games/cartpole.py at N = 50: encoding 8, widest layer 24 (padded), 1538 floats of packed weights, 2 actions, 16 lanes
# per game.  A game's region is 6240 B, the tables and weights every CTA holds 6992 B.
CARTPOLE = dict(N=50, A=2, E=8, maxw=24, blob=1538, G=16, teacher=0)
FIELDS = ("threads", "groups", "ctas_per_sm", "slots", "passes", "smem")


def plan(n, threads=0, **kw):
    from muzero_general_b200 import _lib
    lib = _lib.load_library()
    p = {**CARTPOLE, **H100, **kw}
    out = (C.c_int64 * 6)()
    ok = lib.mz_debug_fc_search_plan(p["N"], p["A"], p["E"], p["maxw"], p["blob"], p["G"], p["teacher"], n, p["sms"],
                                     p["smem_per_sm"], p["reserve"], p["cap"], p["regs"], threads, out)
    return dict(zip(FIELDS, out)) if ok else None


def test_64_thread_ctas_hold_28_games_per_sm():
    """The fixed 64-thread CTA of earlier builds: 4 games next to the tables and weights; shared memory admits 7 CTAs
    per SM (registers would admit 8), so 4096 games take two passes on 132 SMs."""
    p = plan(4096, threads=64)
    assert p == dict(threads=64, groups=4, ctas_per_sm=7, slots=3696, passes=2, smem=6992 + 4 * 6240)


def test_headline_batch_runs_in_one_pass():
    """4096 games on 132 SMs: 32 games per SM, as four 128-thread CTAs (shared memory admits four) or two 256-thread ones
    (whose 2 x 8 warps x 32 lanes x 128 registers fill the register file exactly); equal passes, so the smaller CTA."""
    p = plan(4096)
    assert p == dict(threads=128, groups=8, ctas_per_sm=4, slots=4224, passes=1, smem=6992 + 8 * 6240)
    q = plan(4096, threads=256)
    assert (q["ctas_per_sm"], q["slots"], q["passes"]) == (2, 4224, 1)
    assert 2 * (q["smem"] + 1024) <= H100["smem_per_sm"]
    assert plan(8192)["passes"] == 2 and plan(8192, threads=64)["passes"] == 3


def test_headline_batch_on_148_sms():
    """148 SMs hold 4144 games in 64-thread CTAs already: one pass, the smallest CTA."""
    p = plan(4096, sms=148)
    assert (p["threads"], p["ctas_per_sm"], p["slots"], p["passes"]) == (64, 7, 4144, 1)


@pytest.mark.parametrize("n", [1, 100, 1000, 3696])
def test_smallest_cta_among_equal_pass_counts(n):
    """Batches that 64-thread CTAs already hold in one pass keep them: more, smaller CTAs spread the games over more SMs."""
    p = plan(n)
    assert p["threads"] == 64 and p["passes"] == 1


def test_one_game_past_the_64_thread_wave_moves_to_128_threads():
    assert plan(3697)["threads"] == 128 and plan(3697)["passes"] == 1
    assert plan(4224)["passes"] == 1 and plan(4225)["passes"] == 2


def test_other_sizes():
    """N = 25: a game needs about 3.6 KB, so 64-thread CTAs are register-bound at 8 per SM, 32 games per SM, and keep the
    headline batch in one pass.  G = 32: 8 games per 256-thread CTA, two CTAs, 16 games per SM whatever the CTA size
    (registers bound them all), so the smallest CTA.  The teacher-forced kernel has no weights or hidden states."""
    p = plan(4096, N=25)
    assert (p["threads"], p["ctas_per_sm"], p["passes"]) == (64, 8, 1)
    for n in (1000, 4096):
        p = plan(n, G=32)
        assert p["threads"] == 64 and p["ctas_per_sm"] * p["groups"] == 16
        assert p["passes"] == -(-n // (16 * 132))
    for threads in (64, 128, 256):
        q = plan(4096, G=32, threads=threads)
        assert q["ctas_per_sm"] * threads * 128 == 65536 and q["groups"] == threads // 32
    t = plan(4096, teacher=1, E=1, maxw=4, blob=0)
    assert t["passes"] == 1 and t["smem"] < plan(4096, threads=t["threads"])["smem"]


def test_129_registers_leave_one_256_thread_cta():
    """Eight more registers per thread (the allocation unit) and a 256-thread CTA no longer fits twice (16 games per SM),
    nor four 128-thread ones (24 games per SM): the headline batch is back to two passes, in 64-thread CTAs."""
    assert plan(4096, regs=129, threads=256)["ctas_per_sm"] == 1
    assert plan(4096, regs=129, threads=128)["ctas_per_sm"] == 3
    p = plan(4096, regs=129)
    assert not (p["threads"] == 256 and p["ctas_per_sm"] == 2)
    assert (p["threads"], p["slots"], p["passes"]) == (64, 3696, 2)


def test_a_game_that_does_not_fit_gives_no_plan():
    """N = 2000: one game's tree is 240 KB, beyond the 227 KB a CTA may have; the search then runs step by step."""
    assert plan(4096, N=2000) is None
    assert plan(4096, N=2000, threads=64) is None
    assert plan(4096, threads=48) is None                     # not a whole number of warps
    assert plan(4096, threads=512) is None                    # beyond the kernel's launch bounds
