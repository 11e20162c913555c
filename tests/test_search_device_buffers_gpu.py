"""SearchEngine.search on device tensors hands every search its own output buffer, the next one allocated while the
previous search runs: consecutive searches of one batch size return arrays that keep their own values, each equal to
mz_search's on the same inputs."""
import pytest

from test_search_device_call_gpu import _assert_equal, _engine, _host, _inputs, _mz_search

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [31, 4096])
def test_consecutive_searches_keep_their_own_arrays(n, game_configs):
    cfg = game_configs["cartpole"]
    eng = _engine(cfg)
    kept = []
    for i in range(4):
        inp = _inputs(cfg, n, seed=200 + i)
        kw = dict(add_exploration_noise=True, noise=inp["noise"], game_id=inp["game_id"])
        out = eng.search(obs=inp["obs"], **kw)
        kept.append((out, _mz_search(eng, n, inp["obs"], **kw)))
    assert len({out.visit_counts.data_ptr() for out, _ in kept}) == len(kept)
    for i, (out, ref) in enumerate(kept):
        _assert_equal(_host(out), ref, (n, i))
    eng.close()
