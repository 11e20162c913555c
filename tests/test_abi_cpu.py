"""CPU-side checks of the boundary: the library loads, exports every declared symbol, the
Python structs match the header, and there is no CPU fallback."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def test_library_exports_every_declared_symbol():
    from muzero_general_b200 import _lib
    lib = _lib.load_library()
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    declared = set(re.findall(r"^\s*(?:const\s+)?[a-z0-9_]+\s*\*?\s*(mz_[a-z0-9_]+)\s*\(", header, re.M))
    assert declared, "no prototypes parsed"
    bound = {name for name, _, _ in _lib.SYMBOLS}
    assert declared == bound, (declared ^ bound)
    for name in declared:
        assert hasattr(lib, name)
    assert lib.mz_abi_version() == 2


_PRIM = {"int32_t": 4, "uint32_t": 4, "int64_t": 8, "uint64_t": 8, "double": 8, "float": 4, "uint8_t": 1, "int8_t": 1, "int": 4}


def _header_structs():
    """Parse every `typedef struct X { ... } X;` of include/mzb200.h into [(field, offset, size)] + total size,
    with natural alignment (what gcc / nvcc do for these plain structs)."""
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    consts = {k: int(v) for k, v in re.findall(r"#define\s+(MZ_[A-Z_]+)\s+(\d+)", header)}
    text = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    out = {}
    for name, body in re.findall(r"typedef struct (\w+) \{(.*?)\} \1;", text, flags=re.S):
        off, align_max, fields = 0, 1, []
        for decl in body.split(";"):
            decl = " ".join(decl.split())
            if not decl:
                continue
            m = re.match(r"(?:const )?(?:struct )?(\w+)(\s*\*)?\s*(.*)", decl)
            base, star, rest = m.group(1), m.group(2), m.group(3)
            for item in rest.split(","):
                item = item.strip()
                ptr = bool(star) or item.startswith("*")
                item = item.lstrip("* ")
                am = re.match(r"(\w+)\[(\w+)\]", item)
                count = 1
                if am:
                    item, count = am.group(1), consts.get(am.group(2)) or int(am.group(2))
                size = 8 if ptr else _PRIM[base]
                off = (off + size - 1) // size * size
                fields.append((item, off, size * count))
                off += size * count
                align_max = max(align_max, size)
        out[name] = (fields, (off + align_max - 1) // align_max * align_max)
    return out


def test_ctypes_structs_match_the_header_field_by_field():
    from muzero_general_b200 import _lib
    structs = _header_structs()
    assert {"MzNetDesc", "MzSearchDesc", "MzSearchIO", "MzSelfPlayDesc", "MzSelfPlayStats"} <= set(structs)
    for name, (fields, size) in structs.items():
        cls = getattr(_lib, name)
        assert ctypes.sizeof(cls) == size, (name, ctypes.sizeof(cls), size)
        assert [f[0] for f in cls._fields_] == [f[0] for f in fields], name
        for fname, off, fsize in fields:
            d = getattr(cls, fname)
            assert (d.offset, d.size) == (off, fsize), (name, fname)


def test_integration_doc_stub_matches_the_library():
    """INTEGRATION.md shows the ctypes stub a maintainer would paste: every fenced python block that defines
    Structures is executed and its classes must have the layout of the real binding."""
    from muzero_general_b200 import _lib
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    blocks = [b for b in re.findall(r"```python\n(.*?)```", doc, flags=re.S) if "C.Structure" in b]
    assert blocks, "no ctypes stub found in INTEGRATION.md"
    checked = 0
    for block in blocks:
        # keep the declarations, drop the usage lines that need a GPU / real buffers
        decl = block.split("# ---- usage")[0]
        ns = {}
        exec(decl, ns)
        for name, obj in ns.items():
            if isinstance(obj, type) and issubclass(obj, ctypes.Structure) and obj is not ctypes.Structure:
                real = getattr(_lib, name)
                assert ctypes.sizeof(obj) == ctypes.sizeof(real), name
                assert [(f[0], getattr(obj, f[0]).offset) for f in obj._fields_] == \
                       [(f[0], getattr(real, f[0]).offset) for f in real._fields_], name
                checked += 1
    assert checked >= 3


def test_no_cpu_fallback(game_configs):
    """Without a GPU mz_create must fail loudly rather than compute on the host."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import SearchEngine
    with pytest.raises(_lib.MzError) as e:
        SearchEngine(game_configs["cartpole"], max_games=4)
    assert "no CPU fallback" in str(e.value)


def test_more_than_two_players_rejected(game_configs):
    """self_play.py:429-430 raises NotImplementedError; so does the boundary."""
    import copy
    cfg = copy.deepcopy(game_configs["cartpole"])
    cfg.players = [0, 1, 2]
    from muzero_general_b200.engine import SearchEngine
    with pytest.raises(NotImplementedError):
        SearchEngine(cfg, max_games=1)


def test_bench_conv_flops_agree_with_survey_table():
    """bench.py derives the tensor roofline's algorithmic FLOPs from the network shape; the 3x3 convolutions must account
    for (almost) all of the per-inference FLOPs quoted in SURVEY.md section 8 (the rest are the 1x1 convs and FC heads)."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.dirname(__file__)), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config
    for game, N in (("tictactoe", 50), ("connect4", 200), ("breakout", 50)):
        ns = netspec_from_config(load_game_module(game).MuZeroConfig())
        f0, f1 = bench.NET_FLOPS[game]
        conv = bench.conv3x3_flops(ns, N)
        total = f0 + N * f1
        assert 0.85 * total < conv <= total, (game, conv, total)


def test_small_search_launch_plan():
    """Host-side planner of the fused small-network search (csrc/small_search.cu::small_search_shape): tile sizes fill
    whole waves of SMs, shared memory stays inside the 227 KB a CTA may use, the uniform-weight mapping gets the strides
    that spread 32 rows over 32 banks, and shapes without an instantiated kernel are refused."""
    import ctypes as C
    from muzero_general_b200 import _lib
    lib = _lib.load_library()

    def plan(H, W, Cc, A, n, tower=11664, heads=5000, scratch=868, cap=17, sms=132):
        out = (C.c_int64 * 8)()
        ok = lib.mz_debug_small_search_plan(H, W, Cc, A, n, sms, tower, heads, scratch, cap, out)
        return dict(zip(("P", "CO", "G", "tile", "threads", "smem", "row_stride", "board_stride"), out)) if ok else None

    # TicTacToe, BASELINE batch: 8192 games on 132 SMs -> three even waves of CTAs, one lane group per game, four output channels
    # per thread
    p = plan(3, 3, 16, 9, 8192)
    assert (p["P"], p["CO"], p["G"]) == (3, 4, 16)
    ctas = -(-8192 // p["tile"])
    assert 2.9 < ctas / 132 <= 3.0 and p["tile"] * 16 <= p["threads"] <= 512 and p["threads"] % 32 == 0
    assert p["smem"] <= 227 * 1024
    # bank spreading of the uniform-weight mapping: odd row stride, 32 consecutive rows (board, y) hit 32 different banks
    assert p["row_stride"] % 2 == 1 and p["board_stride"] >= 17 * 5 * p["row_stride"]
    banks = {((r // 3) * p["board_stride"] + (r % 3) * p["row_stride"]) % 32 for r in range(32)}
    assert len(banks) == 32
    # a handful of games: one channel per thread (more threads per board), still one CTA per tile
    q = plan(3, 3, 16, 9, 5)
    assert q["CO"] == 1 and q["tile"] == 1
    # the Breakout configuration's hidden board: 6 x 6 x 16, 4 actions, 128 games on 132 SMs -> one game per CTA
    b = plan(6, 6, 16, 4, 128, tower=21024, heads=8600, scratch=1408)
    assert b["G"] == 4 and b["tile"] == 1 and b["smem"] <= 227 * 1024
    # same board, a large batch: uniform weights with P = W = 6
    b2 = plan(6, 6, 16, 4, 4096, tower=21024, heads=8600, scratch=1408)
    assert (b2["P"], b2["CO"]) == (6, 4) and b2["row_stride"] == 9 and b2["smem"] <= 227 * 1024
    banks = {((r // 6) * b2["board_stride"] + (r % 6) * b2["row_stride"]) % 32 for r in range(32)}
    assert len(banks) == 32
    # not handled: 7 actions (no lane-group instantiation), a 7-wide board, weights beyond shared memory
    assert plan(3, 3, 16, 7, 100) is None
    assert plan(6, 7, 16, 4, 100) is None
    assert plan(3, 3, 16, 9, 100, tower=70000) is None
