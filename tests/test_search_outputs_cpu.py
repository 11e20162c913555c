"""The one-buffer outputs of a device-memory search (engine.output_layout / carve_outputs), checked on CPU tensors: every
SearchOutput array keeps its dtype and shape, starts 16-byte aligned, is contiguous and overlaps no other; each buffer
gets its own arrays."""
import numpy
import pytest

from muzero_general_b200.engine import SearchOutput, carve_outputs, output_layout

FIELDS = ("visit_counts", "root_value", "root_predicted_value", "max_tree_depth", "tie_count", "root_priors", "value_range")


def _expected(n, A):
    import torch
    return {"visit_counts": ((n, A), torch.int32), "root_value": ((n,), torch.float64),
            "root_predicted_value": ((n,), torch.float32), "max_tree_depth": ((n,), torch.int32),
            "tie_count": ((n,), torch.int32), "root_priors": ((n, A), torch.float64), "value_range": ((n, 2), torch.float64)}


@pytest.mark.parametrize("n", [1, 3, 31, 4096, 4224])
@pytest.mark.parametrize("A", [2, 3, 7, 9, 256])
def test_layout_and_views(n, A):
    import torch
    fields, nbytes = output_layout(n, A)
    assert len(fields) == len(FIELDS) and nbytes % 16 == 0
    offsets = [f[3] for f in fields]
    assert offsets[0] == 0 and all(o % 16 == 0 for o in offsets) and offsets == sorted(offsets)
    buf = torch.empty(nbytes // 8, dtype=torch.float64)
    out = carve_outputs(buf, fields)
    assert isinstance(out, SearchOutput) and out.trace is None and out.device_ms == 0.0
    want = _expected(n, A)
    spans = []
    for name, off in zip(FIELDS, offsets):
        t = getattr(out, name)
        shape, dtype = want[name]
        assert tuple(t.shape) == shape and t.dtype == dtype and t.is_contiguous(), name
        assert t.data_ptr() == buf.data_ptr() + off and t.data_ptr() % 16 == 0, name
        spans.append((off, off + t.numel() * t.element_size()))
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a1 <= b0
    assert spans[-1][1] <= nbytes
    # the arrays are what the views say: writes through one never reach another
    for i, name in enumerate(FIELDS):
        getattr(out, name).fill_(i + 1)
    for i, name in enumerate(FIELDS):
        assert (getattr(out, name) == i + 1).all(), name


def test_each_buffer_gets_its_own_arrays():
    import torch
    fields, nbytes = output_layout(31, 2)
    a = carve_outputs(torch.zeros(nbytes // 8, dtype=torch.float64), fields)
    b = carve_outputs(torch.zeros(nbytes // 8, dtype=torch.float64), fields)
    a.visit_counts.fill_(7)
    b.visit_counts.fill_(3)
    assert (a.visit_counts == 7).all() and (b.visit_counts == 3).all()
    assert numpy.array_equal(a.root_value.numpy(), numpy.zeros(31))
