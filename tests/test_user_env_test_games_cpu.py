"""Test-mode games of user environments on the host alone: sources with MZ_ENV_EXPERT compile an expert wrapper without
spills (mz_debug_user_env_expert_compile), sources without it compile none and the same reset and step wrappers, a
source that defines the macro but not the function is refused naming it, and SelfPlay.play_test_games picks its route
for every opponent, with and without an expert and with and without config.host_env_device_loop."""
import pytest

from conftest import weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from user_env_contract_games import CASES
from user_env_expert_sources import SOURCES, contract_expert_source
from user_env_sources import SOURCES as PLAIN_SOURCES

MZ_EINVAL = -1

EXPERT_SOURCES = dict({name: src for name, (src, _, _) in SOURCES.items()},
                      **{"contract_" + c.name: contract_expert_source(c) for c in CASES.values() if c.P == 2})


@pytest.mark.parametrize("name", sorted(EXPERT_SOURCES))
def test_expert_sources_compile_an_expert_wrapper_without_spills(name):
    from muzero_general_b200.engine import debug_user_env_expert_compile
    rc, log, info = debug_user_env_expert_compile(EXPERT_SOURCES[name])
    assert rc == 0, log
    assert info["expert"], info
    for kernel in ("reset", "step", "expert_kernel"):
        regs, frame, spill_stores, spill_loads = info[kernel]
        assert 0 < regs <= 255 and frame >= 0, (kernel, info)
        assert spill_stores == 0 and spill_loads == 0, (kernel, info)
    assert "Compiling entry function 'mz_user_env_expert'" in log


@pytest.mark.parametrize("name", sorted(PLAIN_SOURCES))
def test_sources_without_the_macro_compile_no_expert_and_the_same_wrappers(name):
    from muzero_general_b200.engine import debug_user_env_compile, debug_user_env_expert_compile
    rc, log, info = debug_user_env_expert_compile(PLAIN_SOURCES[name][0])
    assert rc == 0, log
    assert not info["expert"] and info["expert_kernel"] == (-1, -1, -1, -1), info
    assert "mz_user_env_expert" not in log
    rc0, log0, info0 = debug_user_env_compile(PLAIN_SOURCES[name][0])
    report = lambda text: [line for line in text.splitlines() if "Compile time" not in line]   # noqa: E731
    assert rc0 == 0 and report(log0) == report(log)
    assert {k: info[k] for k in info0} == info0


def test_the_expert_does_not_change_the_reset_and_step_wrappers():
    """The same rules with and without the expert: ptxas reports the same reset and step wrappers."""
    from muzero_general_b200.engine import debug_user_env_expert_compile
    _, _, plain = debug_user_env_expert_compile(PLAIN_SOURCES["tictactoe"][0])
    _, _, expert = debug_user_env_expert_compile(SOURCES["tictactoe"][0])
    assert (plain["reset"], plain["step"]) == (expert["reset"], expert["step"])


def test_the_macro_without_the_function_is_refused_naming_it():
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_user_env_compile, debug_user_env_expert_compile
    src = SOURCES["tictactoe"][0].replace("mz_env_expert(", "renamed_expert(")
    for compile_ in (debug_user_env_expert_compile, debug_user_env_compile):
        rc, _, _ = compile_(src)
        assert rc == MZ_EINVAL
        msg = _lib.load_library().mz_last_error(None).decode()
        assert "MZ_ENV_EXPERT" in msg and "mz_env_expert" in msg, msg


# ------------------------------------------------------------------------------------------ route of play_test_games
class Routed(Exception):
    """Raised by the stand-ins for the loops: which loop play_test_games built, with which opponent."""


def _fake_user_loop(engine, source, state_bytes, obs_shape, max_moves, opponent="self", muzero_player=0, **kw):
    # the library's answer to EXPERT on a source without mz_env_expert (mz_selfplay_begin_user_vs: MZ_EUNSUPPORTED)
    if opponent == "expert" and "#define MZ_ENV_EXPERT" not in source:
        raise NotImplementedError("mz_selfplay_begin_user_vs: the source has no expert opponent")
    raise Routed("device-user-env", opponent, muzero_player)


def _fake_host_loop(*args, opponent="self", muzero_player=0, **kw):
    raise Routed("device-host-env", opponent, muzero_player)


@pytest.fixture()
def fakes(monkeypatch):
    monkeypatch.setattr(sp, "SearchEngine", FakeSearchEngine)
    monkeypatch.setattr(sp, "UserEnvSelfPlayLoop", _fake_user_loop)
    monkeypatch.setattr(sp, "HostEnvSelfPlayLoop", _fake_host_loop)


def _route(source, opponent, host_env_device_loop):
    mod = load_game_module("tictactoe")
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.host_env_device_loop = 4, "philox", host_env_device_loop
    Game = type("UserGame", (mod.Game,), dict(DEVICE_ENV=None, DEVICE_SOURCE=source, DEVICE_STATE_BYTES=10))
    w = sp.SelfPlay({"weights": weights_for("tictactoe", netspec_from_config(cfg))}, Game, cfg, seed=0)
    assert w.loop_path == "device-user-env"
    try:
        w.play_test_games(3, opponent, 1)
    except Routed as r:
        assert r.args[1:] == (opponent, 1)
        return r.args[0]
    except NotImplementedError as e:
        return "refused: " + str(e)
    raise AssertionError("play_test_games built no loop")


@pytest.mark.parametrize("host_env_device_loop", [False, True])
@pytest.mark.parametrize("with_expert", [False, True])
def test_route_of_test_games(fakes, with_expert, host_env_device_loop):
    """"self" and "random" play on the user environment; "expert" too when the source has one, else the routes test
    games had before (the host-stepped loop with host_env_device_loop, else NotImplementedError naming play_game);
    "human" keeps those routes."""
    source = SOURCES["tictactoe"][0] if with_expert else PLAIN_SOURCES["tictactoe"][0]
    before = "device-host-env" if host_env_device_loop else "refused"
    assert _route(source, "self", host_env_device_loop) == "device-user-env"
    assert _route(source, "random", host_env_device_loop) == "device-user-env"
    got = _route(source, "expert", host_env_device_loop)
    assert got.startswith("device-user-env" if with_expert else before), got
    if got.startswith("refused"):
        assert "MZ_ENV_EXPERT" in got or "expert" in got
    got = _route(source, "human", host_env_device_loop)
    assert got.startswith(before), got
    if got.startswith("refused"):
        assert "play_game" in got
