"""ORACLE support: compact, exact encodings for fixtures whose arrays grow with the action space
(``oracle/gen_golden_wide.py`` writes them, the tests read them back into the plain lists the other fixtures hold).

* a list of floats becomes ``{"f32": base64}`` when every value is an fp32 value, else ``{"f64": base64}`` (little
  endian); decoding gives the same Python floats, bit for bit
* a subset of ``range(n)`` that misses few members becomes ``{"n": n, "missing": [...]}``
* a board observation ``[stones of +1, stones of -1, side plane]`` becomes the two stone lists and the side
"""
import base64

import numpy


def pack_floats(values):
    a64 = numpy.asarray(values, dtype="<f8")
    a32 = a64.astype("<f4")
    if numpy.array_equal(a32.astype("<f8"), a64) and not numpy.signbit(a64[a64 == 0]).any():
        return {"f32": base64.b64encode(a32.tobytes()).decode()}
    return {"f64": base64.b64encode(a64.tobytes()).decode()}


def unpack_floats(packed):
    (kind, text), = packed.items()
    a = numpy.frombuffer(base64.b64decode(text), dtype="<f4" if kind == "f32" else "<f8")
    return [float(x) for x in a]


def pack_subset(members, n):
    have = set(members)
    assert list(members) == sorted(have) and have <= set(range(n))
    return {"n": n, "missing": [k for k in range(n) if k not in have]}


def unpack_subset(packed):
    missing = set(packed["missing"])
    return [k for k in range(packed["n"]) if k not in missing]


def pack_board(obs):
    o = numpy.asarray(obs)
    cells = o.shape[1] * o.shape[2]
    flat = o.reshape(3, cells)
    side = int(flat[2, 0])
    assert set(numpy.unique(flat[:2])) <= {0, 1} and (flat[2] == side).all()
    return {"x": numpy.nonzero(flat[0])[0].tolist(), "o": numpy.nonzero(flat[1])[0].tolist(), "side": side}


def unpack_board(packed, cells):
    """The flat int8 list [plane 0 | plane 1 | plane 2] of the other env_*.json fixtures."""
    flat = numpy.zeros((3, cells), numpy.int8)
    flat[0, packed["x"]] = 1
    flat[1, packed["o"]] = 1
    flat[2] = packed["side"]
    return flat.ravel().tolist()
