"""SearchEngine.search on device tensors goes through mz_search_device (one output buffer, the handle's prepared fused
launch).  Its arrays must be mz_search's on the same inputs, bit for bit, whatever the batch, the optional inputs and
the order of the calls."""
import ctypes as C

import numpy
import pytest

from muzero_general_b200 import _lib

pytestmark = pytest.mark.gpu

FIELDS = ("visit_counts", "root_value", "root_predicted_value", "max_tree_depth", "tie_count", "root_priors", "value_range")
MAX_GAMES, N_SIM = 4224, 50


def _engine(cfg, max_games=MAX_GAMES, weights_seed=0):
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    eng = SearchEngine(cfg, max_games=max_games, num_simulations=N_SIM)
    eng.load_weights(synthetic_weights(netspec_from_config(cfg), weights_seed))
    return eng


def _inputs(cfg, n, seed):
    import torch
    rs = numpy.random.RandomState(seed)
    A = len(cfg.action_space)
    legal = (rs.rand(n, A) < 0.7).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    t = lambda a: torch.from_numpy(a).cuda()
    return dict(obs=t(rs.uniform(-0.05, 0.05, size=(n, 4)).astype(numpy.float32)),
                noise=t(rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)),
                game_id=t(rs.randint(0, 1 << 40, n).astype(numpy.int64)),
                legal_mask=t(legal), first_index=t(rs.randint(0, A, n).astype(numpy.int32)))


def _mz_search(eng, n, obs, add_exploration_noise=False, noise=None, game_id=None, legal_mask=None, first_index=None):
    """The same search through mz_search with MZ_MEM_DEVICE (what SearchEngine.search called before)."""
    import torch
    A, dev = eng.A, obs.device
    io = _lib.MzSearchIO()
    io.n_games, io.mem = n, _lib.MZ_MEM_DEVICE
    io.add_exploration_noise = int(bool(add_exploration_noise))
    p = lambda x: None if x is None else x.data_ptr()
    io.obs, io.noise, io.game_id, io.legal_mask, io.first_index = p(obs), p(noise), p(game_id), p(legal_mask), p(first_index)
    out = [torch.full((n, A), -7, dtype=torch.int32, device=dev), torch.full((n,), -7.0, dtype=torch.float64, device=dev),
           torch.full((n,), -7.0, dtype=torch.float32, device=dev), torch.full((n,), -7, dtype=torch.int32, device=dev),
           torch.full((n,), -7, dtype=torch.int32, device=dev), torch.full((n, A), -7.0, dtype=torch.float64, device=dev),
           torch.full((n, 2), -7.0, dtype=torch.float64, device=dev)]
    (io.visit_counts, io.root_value, io.root_predicted_value, io.max_tree_depth, io.tie_count, io.root_priors,
     io.value_range) = (t.data_ptr() for t in out)
    eng._check(eng.lib.mz_search(eng._h, C.byref(io)))
    return {f: t.cpu().numpy() for f, t in zip(FIELDS, out)}


def _host(out):
    return {f: getattr(out, f).cpu().numpy() for f in FIELDS}


def _assert_equal(a, b, what):
    for f in FIELDS:
        assert a[f].dtype == b[f].dtype and a[f].shape == b[f].shape, (what, f)
        assert numpy.array_equal(a[f], b[f]), (what, f)


OPTIONAL = [(), ("game_id",), ("legal_mask",), ("first_index",), ("game_id", "legal_mask", "first_index")]


@pytest.mark.parametrize("n", [1, 31, 4096, 4224])
@pytest.mark.parametrize("noise", ["off", "given", "device"])
def test_device_call_matches_mz_search(n, noise, game_configs):
    cfg = game_configs["cartpole"]
    eng = _engine(cfg)
    inp = _inputs(cfg, n, seed=n)
    for opt in OPTIONAL:
        kw = {k: inp[k] for k in opt}
        if noise != "off":
            kw["add_exploration_noise"] = True
        if noise == "given":
            kw["noise"] = inp["noise"]
        l0 = eng.launch_count
        new = eng.search(obs=inp["obs"], **kw)
        assert eng.launch_count == l0 + 1                          # one fused launch
        assert new.device_ms > 0.0 and new.device_ms == eng.last_search_ms
        old = _mz_search(eng, n, inp["obs"], **kw)
        _assert_equal(_host(new), old, (n, noise, opt))
        assert int(new.visit_counts.sum()) == n * N_SIM
    assert eng.fc_prepared["games"] == n
    eng.close()


def test_changing_batch_reprepares_and_earlier_outputs_keep_their_values(game_configs):
    """Searches over 4096, 31, 4224, 1 and 4096 games on one handle, each against mz_search: the prepared launch follows
    the batch (grid included), and every SearchOutput returned so far still holds its own arrays."""
    cfg = game_configs["cartpole"]
    eng = _engine(cfg)
    kept = []
    for i, n in enumerate((4096, 31, 4224, 1, 4096)):
        inp = _inputs(cfg, n, seed=100 + i)
        out = eng.search(obs=inp["obs"], add_exploration_noise=True, noise=inp["noise"], game_id=inp["game_id"])
        assert eng.fc_prepared["games"] == n
        grid = eng.last_fc_launch["grid"]
        ref = _mz_search(eng, n, inp["obs"], add_exploration_noise=True, noise=inp["noise"], game_id=inp["game_id"])
        _assert_equal(_host(out), ref, n)
        kept.append((out, ref, grid))
    assert kept[0][2] != kept[1][2] and kept[1][2] != kept[2][2]
    for out, ref, _ in kept:
        _assert_equal(_host(out), ref, "kept")
    eng.close()


@pytest.mark.parametrize("switch", ["MZ_FC_GENERIC", "MZ_FC_SELECT_LEVELS"])
def test_ab_switches_take_effect_on_a_new_handle(switch, monkeypatch, game_configs):
    """MZ_FC_GENERIC=1 picks the descriptor-walking instantiation, MZ_FC_SELECT_LEVELS=1 one tree level per round; the
    device call under either gives the default's arrays."""
    cfg = game_configs["cartpole"]
    n = 1000
    inp = _inputs(cfg, n, seed=7)
    kw = dict(obs=inp["obs"], add_exploration_noise=True, noise=inp["noise"], legal_mask=inp["legal_mask"])
    monkeypatch.delenv("MZ_FC_GENERIC", raising=False)
    monkeypatch.delenv("MZ_FC_SELECT_LEVELS", raising=False)
    eng = _engine(cfg, max_games=n)
    base = _host(eng.search(**kw))
    default = eng.fc_prepared
    eng.close()
    assert default["fixed_shape"] == 1 and default["generic"] == 0 and default["select_levels"] > 1
    monkeypatch.setenv(switch, "1")
    eng = _engine(cfg, max_games=n)
    out = _host(eng.search(**kw))
    prep = eng.fc_prepared
    eng.close()
    if switch == "MZ_FC_GENERIC":
        assert prep["generic"] == 1 and prep["fixed_shape"] == 0
    else:
        assert prep["one_level"] == 1 and prep["select_levels"] == 1
    _assert_equal(out, base, switch)


def test_loading_weights_drops_the_prepared_launch(game_configs):
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    cfg = game_configs["cartpole"]
    eng = _engine(cfg, max_games=64)
    inp = _inputs(cfg, 64, seed=3)
    eng.search(obs=inp["obs"])
    assert eng.fc_prepared is not None
    eng.load_weights(synthetic_weights(netspec_from_config(cfg), 1))
    assert eng.fc_prepared is None
    out = _host(eng.search(obs=inp["obs"], game_id=inp["game_id"]))
    _assert_equal(out, _mz_search(eng, 64, inp["obs"], game_id=inp["game_id"]), "reloaded")
    eng.close()


def test_each_enqueue_needs_its_wait(game_configs):
    """mz_search_device refuses a second search before the first one's wait, and a wait needs a search."""
    cfg = game_configs["cartpole"]
    eng = _engine(cfg, max_games=32)
    inp = _inputs(cfg, 32, seed=5)
    ref = _host(eng.search(obs=inp["obs"]))
    assert eng.lib.mz_search_device_wait(eng._h, eng._dio_ref) == _lib.MZ_ESTATE
    out = eng.search(obs=inp["obs"])
    io = eng._dio                                  # the pointers of that call are still in the engine's struct
    assert eng.lib.mz_search_device(eng._h, eng._dio_ref) == 0
    assert eng.lib.mz_search_device(eng._h, eng._dio_ref) == _lib.MZ_ESTATE
    assert eng.lib.mz_search_device_wait(eng._h, eng._dio_ref) == 0 and io.device_ms > 0.0
    _assert_equal(_host(out), ref, "again")
    eng.close()
