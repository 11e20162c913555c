"""User environments on the host alone: the sample sources compile for sm_90a through mz_debug_user_env_compile (NVRTC
needs no GPU) without spills, a source that does not compile or lacks one of the contract's functions is refused with
its reason, the ABI's struct matches the header and INTEGRATION.md's stub, and SelfPlay picks the "device-user-env"
route only where it should."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from user_env_sources import SOURCES

MZ_EINVAL = -1


@pytest.mark.parametrize("name", sorted(SOURCES))
def test_sample_sources_compile_without_spills(name):
    from muzero_general_b200.engine import debug_user_env_compile
    rc, log, info = debug_user_env_compile(SOURCES[name][0])
    assert rc == 0, log
    assert info["nvrtc_version"] >= 12000
    for kernel in ("reset", "step"):
        regs, frame, spill_stores, spill_loads = info[kernel]
        assert 0 < regs <= 255 and frame >= 0, (kernel, info)
        assert spill_stores == 0 and spill_loads == 0, (kernel, info)
    assert "for 'sm_90a'" in log


def test_a_syntax_error_names_its_line():
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_user_env_compile
    src = SOURCES["simple_grid"][0]
    lines = src.split("\n")
    bad = next(i for i, line in enumerate(lines) if "++s->col;" in line)
    lines[bad] = lines[bad].replace("++s->col;", "++s->col")
    rc, log, _ = debug_user_env_compile("\n".join(lines))
    assert rc == MZ_EINVAL
    # the user's own line numbers: the prelude is pre-included, not pasted in front; the parser reports the missing
    # ";" at the next token, on the line after
    m = re.search(r"user_env_source\.cu\((\d+)\): error", log)
    assert m and int(m.group(1)) in (bad + 1, bad + 2), log
    assert "error" in _lib.load_library().mz_last_error(None).decode()


@pytest.mark.parametrize("missing", ["mz_env_step", "mz_env_reset"])
def test_a_source_without_a_contract_function_is_refused(missing):
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_user_env_compile
    src = SOURCES["tictactoe"][0].replace(missing + "(", "renamed_" + missing + "(")
    rc, _, _ = debug_user_env_compile(src)
    assert rc == MZ_EINVAL
    msg = _lib.load_library().mz_last_error(None).decode()
    assert "does not define" in msg and missing in msg, msg


def test_user_env_desc_matches_the_header_and_the_integration_stub():
    from muzero_general_b200 import _lib
    from test_abi_cpu import _header_structs
    fields, size = _header_structs()["MzUserEnvDesc"]
    cls = _lib.MzUserEnvDesc
    assert ctypes.sizeof(cls) == size
    assert [(f, getattr(cls, f).offset, getattr(cls, f).size) for f, _ in cls._fields_] == fields
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    stubs = [b for b in re.findall(r"```python\n(.*?)```", doc, flags=re.S) if "class MzUserEnvDesc" in b]
    assert len(stubs) == 1
    ns = {}
    exec(stubs[0].split("# ---- usage")[0], ns)
    assert ctypes.sizeof(ns["MzUserEnvDesc"]) == size
    assert [(f[0], getattr(ns["MzUserEnvDesc"], f[0]).offset) for f in ns["MzUserEnvDesc"]._fields_] == \
           [(f, off) for f, off, _ in fields]
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    assert int(re.search(r"#define MZ_ENV_USER (\d+)", header).group(1)) == _lib.MZ_ENV_USER
    assert int(re.search(r"#define MZ_USER_ENV_MAX_STATE_BYTES (\d+)", header).group(1)) == _lib.MZ_USER_ENV_MAX_STATE_BYTES


def test_loop_path_of_user_environments():
    """DEVICE_SOURCE plays on the device with philox draws and device_envs on, unless a built-in device environment is in
    use; bundled plug-ins have none, so their routes do not change."""
    from muzero_general_b200 import self_play as sp
    from muzero_general_b200.games import load_game_module

    def path(Game, rng_mode="philox", **cfg):
        w = sp.SelfPlay.__new__(sp.SelfPlay)
        w.Game, w.rng_mode = Game, rng_mode
        w.config = type("Cfg", (), cfg)()
        return w.loop_path

    base = load_game_module("simple_grid").Game
    user = type("UserGame", (base,), dict(DEVICE_ENV=None, DEVICE_SOURCE=SOURCES["simple_grid"][0], DEVICE_STATE_BYTES=8))
    assert path(user) == "device-user-env"
    assert path(user, host_env_device_loop=True) == "device-user-env"
    assert path(user, rng_mode="numpy") == "host"
    assert path(user, device_envs=False) == "host"
    assert path(user, device_envs=False, host_env_device_loop=True) == "device-host-env"
    both = type("BothGame", (base,), dict(DEVICE_SOURCE=SOURCES["simple_grid"][0], DEVICE_STATE_BYTES=8))
    assert path(both) == "device"
    for name in ("cartpole", "tictactoe", "connect4", "gomoku", "twentyone", "simple_grid", "gridworld", "breakout",
                 "atari"):
        assert getattr(load_game_module(name).Game, "DEVICE_SOURCE", None) is None, name
