"""CTA size of the fused FC search on the device: the headline batch is resident in one wave, and the planned launch
computes exactly what the fixed 64-thread CTAs of earlier builds computed (MZ_FC_THREADS=64), on the fixed-shape and the
generic network path, at batch sizes on both sides of each CTA size's wave."""
import numpy
import pytest

from conftest import golden_npz

pytestmark = pytest.mark.gpu

NS = (1, 100, 3169, 4096, 4225, 8192)
N_SIM = 50


def _engine(monkeypatch, cfg, spec, weights, threads, max_games):
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.netspec import synthetic_weights
    if threads:
        monkeypatch.setenv("MZ_FC_THREADS", str(threads))
    else:
        monkeypatch.delenv("MZ_FC_THREADS", raising=False)
    eng = SearchEngine(cfg, max_games=max_games, num_simulations=N_SIM)
    eng.load_weights(synthetic_weights(spec, 0) if weights == "synthetic" else golden_npz("weights_cartpole_pretrained.npz"))
    return eng


def _inputs(spec, cfg, n, seed):
    rs = numpy.random.RandomState(seed)
    obs = rs.uniform(-0.05, 0.05, size=(n, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * spec.action_space, size=n)
    return dict(obs=obs, add_exploration_noise=True, noise=noise, game_id=numpy.arange(n, dtype=numpy.int64))


def test_headline_batch_is_resident_in_one_wave(monkeypatch, game_configs):
    import torch
    from muzero_general_b200.netspec import netspec_from_config
    cfg = game_configs["cartpole"]
    spec = netspec_from_config(cfg)
    n = 4096
    eng = _engine(monkeypatch, cfg, spec, "synthetic", None, n)
    eng.search(**_inputs(spec, cfg, n, 100))
    info = eng.last_fc_launch
    eng.close()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert info is not None and info["group"] == 16
    assert info["ctas_per_sm"] * (info["block"] // info["group"]) * sms >= n
    assert info["grid"] * (info["block"] // info["group"]) >= n


@pytest.mark.parametrize("G", [16, 32])
@pytest.mark.parametrize("weights", ["synthetic", "pretrained"])
def test_planned_cta_size_is_bit_identical_to_64_threads(G, weights, monkeypatch, game_configs):
    from muzero_general_b200.netspec import netspec_from_config
    cfg = game_configs["cartpole"]
    spec = netspec_from_config(cfg)
    monkeypatch.setenv("MZ_FC_GROUP", str(G))
    planned = _engine(monkeypatch, cfg, spec, weights, None, max(NS))
    fixed = _engine(monkeypatch, cfg, spec, weights, 64, max(NS))
    kw = _inputs(spec, cfg, max(NS), 31 * G + len(weights))
    blocks = set()
    for generic in ("0", "1"):
        monkeypatch.setenv("MZ_FC_GENERIC", generic)
        for n in NS:
            args = {k: (v[:n] if isinstance(v, numpy.ndarray) else v) for k, v in kw.items()}
            outs = []
            for eng in (planned, fixed):
                n0 = eng.launch_count
                outs.append(eng.search(trace=True, trace_depth=N_SIM + 1, **args))
                assert eng.launch_count == n0 + 1                 # one fused launch, no step-wise fallback
            assert fixed.last_fc_launch["block"] == 64
            blocks.add(planned.last_fc_launch["block"])
            a, b = outs
            for f in ("visit_counts", "root_value", "root_predicted_value", "max_tree_depth", "tie_count", "root_priors",
                      "value_range"):
                assert numpy.array_equal(getattr(a, f), getattr(b, f)), (generic, n, f)
            for f in a.trace:
                assert numpy.array_equal(a.trace[f], b.trace[f]), (generic, n, "trace", f)
            assert int(a.visit_counts.sum()) == n * N_SIM
    planned.close()
    fixed.close()
    # G = 16: 64-thread CTAs for the small batches, larger ones for the rest.  G = 32: registers hold every CTA size to
    # 16 games per SM, so the plan keeps 64 threads throughout.
    assert 64 in blocks and (len(blocks) > 1) == (G == 16)


def test_trace_actions_are_zero_past_each_leaf(monkeypatch, game_configs):
    """A traced search's actions past each simulation's depth read 0, also where the handle's device trace buffer still
    holds an earlier search's paths: the second search keeps 13 actions per path instead of 51, so it reuses the
    buffer with every path at another offset (and the buffer is copied back whole)."""
    from muzero_general_b200.netspec import netspec_from_config
    cfg = game_configs["cartpole"]
    spec = netspec_from_config(cfg)
    n = 256
    eng = _engine(monkeypatch, cfg, spec, "synthetic", None, n)
    runs = [eng.search(trace=True, trace_depth=D, **_inputs(spec, cfg, n, seed)) for seed, D in ((1, N_SIM + 1), (2, 13))]
    eng.close()
    assert runs[0].trace["actions"].any()
    for out in runs:
        depth, actions = out.trace["depth"], out.trace["actions"]
        past = numpy.arange(actions.shape[2])[None, None, :] >= depth[:, :, None]
        assert past.any() and not actions[past].any(), int(numpy.count_nonzero(actions[past]))
