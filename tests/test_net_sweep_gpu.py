"""Every network route of tests/netcases.py against the fp64 oracle (oracle/net.py with dtype=torch.float64): initial and
recurrent inference at batch sizes that cross the launch and tile boundaries, and the network outputs a search consumes
(gathered parent states, action planes from the tree, pool slots, partitioned replay, the fused small search).

Tolerance rule for the fp32-grade routes (FC, CUDA-core towers, x3 towers), per sample and per output quantity:

    max|dev - ref64| <= K * max|ref32 - ref64| + FLOOR * max(1, max|ref64|)

ref32 is the fp32 oracle (bit-identical to the reference), so its own error sets the scale, and it goes through the same
min-max rescale amplification as the kernels.  Scalars (value, reward) and priors are functions of logits: their budget
adds the first-order sensitivity to the logits' budget (support_to_scalar: dh^-1/dx * E|k - x|; softmax: 2 max p).
K and FLOOR were set on the CUDA-core routes of the first sweep on an H100 (worst ratio printed per case, see DESIGN.md
section 3.6) with a margin of about 3x.  The x3 towers keep 22 significand bits of each operand (x_h and x_l, 11 each)
and drop the x_l * w_l product, so their unit error is a few times fp32's: their budget is K_X3 = 8 K, FLOOR_X3 =
8 FLOOR (the first sweep measured up to 3.5 K).  The fp16 tower mode keeps the absolute bounds of test_resnet_gpu.py,
measured against fp64 (priors: twice the logits bound, softmax's sensitivity); the boards where the fp16 error is larger
have their own bounds in FP16_CASE, each next to the figure measured on an H100."""
import numpy
import pytest
import torch

from netcases import BY_NAME, CASES, SEARCH_CASES, case_spec, edge_weights, make_config
from oracle.net import OracleNet, support_to_scalar

pytestmark = pytest.mark.gpu

K = 16.0
EPS32 = float(numpy.finfo(numpy.float32).eps)
FLOOR = 64 * EPS32
X3 = 8.0
FP16 = dict(logits=5e-3, hidden_max=1e-1, hidden_q999=1.5e-2, scalar=3e-2)
# boards where the fp16 towers' error exceeds the Connect4 bounds, measured on one H100 SXM (700 W), bound ~1.3x that:
FP16_CASE = {
    # one row of 7 positions: channel ranges over the board are small and the rescale amplifies the fp16 error; measured
    # logits 1.51e-2, hidden 0.314 (99.9 %: 3.6e-3), value 3.27e-2
    "tc_1x7": dict(logits=2e-2, hidden_max=4e-1, scalar=4.5e-2),
    # no residual blocks: a ReLU'd channel of sample 1184 spans only 3.2e-3 over the board, so the rescale multiplies the
    # fp16 stem's error by ~300 there; measured hidden 0.176 (99.9 %: 1.0e-3), logits 3.3e-3
    "tc_6x7_b0": dict(hidden_max=2.5e-1),
}

BATCHES = (1, 2, 31, 33, 131, 132, 133)
TC_BATCHES = BATCHES + (593, 1185, 2369)          # x3: > 592 boards per launch; fp16: resident -> streaming -> per conv
BOUNDARIES = (32, 64, 128, 132, 264, 592, 1184, 1185, 1776, 2368)


def _rows(n, A, seed):
    rs = numpy.random.RandomState(seed + n)
    rows = {0, n - 1, min(A - 1, n - 1)}
    for b in BOUNDARIES:
        rows |= {r for r in (b - 1, b) if r < n}
    rows |= set(int(x) for x in rs.randint(0, n, 3))
    return sorted(rows)


def _h_inv_slope(x):
    """d/dx of support_to_scalar's inverse h-transform, in fp64."""
    eps = 0.001
    root = numpy.sqrt(1 + 4 * eps * (numpy.abs(x) + 1 + eps))
    return 2 * ((root - 1) / (2 * eps)) / root


class Ref:
    """fp32 and fp64 oracle outputs of chosen rows, as numpy float64, with the per-row budgets of the tolerance rule."""

    def __init__(self, spec, w):
        self.spec = spec
        self.o32, self.o64 = OracleNet(spec, w), OracleNet(spec, w, torch.float64)

    def _pack(self, r32, r64, recurrent):
        S = self.spec.support_size
        out = {}
        names = ("value_logits", "reward_logits", "policy_logits", "hidden")
        for k, a, b in zip(names, r32, r64):
            out[k] = (a.double().numpy().reshape(len(a), -1), b.numpy().reshape(len(b), -1))
        for k, lk in (("value", "value_logits"), ("reward", "reward_logits")):
            if k == "reward" and not recurrent:
                continue
            a, b = r32[names.index(lk)], r64[names.index(lk)]
            s64 = support_to_scalar(b, S, torch.float64).numpy()[:, 0]
            p = torch.softmax(b, 1).numpy()
            ks = numpy.arange(-S, S + 1)
            x = (p * ks).sum(1)
            out[k] = (support_to_scalar(a, S).double().numpy()[:, 0], s64)
            out[k + "_sens"] = _h_inv_slope(x) * (p * numpy.abs(ks[None] - x[:, None])).sum(1)
        out["priors"] = (torch.softmax(r32[2], 1).double().numpy(), torch.softmax(r64[2], 1).numpy())
        return out

    def initial(self, obs):
        obs = torch.from_numpy(numpy.ascontiguousarray(obs, numpy.float32))
        if self.spec.kind != 0:
            obs = obs.reshape((len(obs), self.spec.in_channels) + tuple(self.spec.obs_shape[1:]))
        return self._pack(self.o32.initial_inference(obs), self.o64.initial_inference(obs), False)

    def recurrent(self, hidden, action):
        h = torch.from_numpy(numpy.ascontiguousarray(hidden, numpy.float32)).reshape((len(hidden),) + self._hshape())
        a = torch.from_numpy(numpy.asarray(action, numpy.int64).reshape(-1, 1))
        return self._pack(self.o32.recurrent_inference(h, a), self.o64.recurrent_inference(h, a), True)

    def _hshape(self):
        if self.spec.kind == 0:
            return (self.spec.encoding,)
        return (self.spec.channels,) + tuple(self.spec.hidden_hw)


class Judge:
    """Applies the tolerance rule and keeps the worst error / budget ratio of a case."""

    def __init__(self, name, mode=None, case=None):
        self.name, self.fp16, self.worst, self.where = name, mode == "fp16", 0.0, ""
        self.k, self.floor = (K * X3, FLOOR * X3) if mode == "x3" else (K, FLOOR)
        # fp16: absolute bounds, checked at finish() over everything the case saw (largest error per kind + where)
        self.fp16_bounds = {**FP16, **FP16_CASE.get(case, {})}
        self.fp16_max = {k: (0.0, "") for k in ("logits", "priors", "hidden", "scalar")}
        self.fp16_hidden = []

    def _fp16(self, kind, err, where):
        if err > self.fp16_max[kind][0]:
            self.fp16_max[kind] = (err, where)

    def _ratio(self, err, budget, where):
        r = err / budget
        if r > self.worst:
            self.worst, self.where = r, where
        assert err <= budget, f"{self.name} {where}: error {err:.3e} > budget {budget:.3e}"

    def logit_budget(self, ref, k, i):
        a, b = ref[k][0][i], ref[k][1][i]
        fin = numpy.isfinite(b)
        return self.k * numpy.abs(a[fin] - b[fin]).max(initial=0.0) + self.floor * max(1.0, numpy.abs(b[fin]).max(initial=0.0))

    def vector(self, what, dev, ref, k, i):
        """dev: the device's row; ref[k] = (ref32 rows, ref64 rows); row i."""
        a, b = ref[k][0][i], ref[k][1][i]
        dev = numpy.asarray(dev, numpy.float64).reshape(-1)
        fin = numpy.isfinite(b)
        assert numpy.array_equal(numpy.isfinite(dev), fin), f"{self.name} {what}: non-finite entries differ"
        err = numpy.abs(dev[fin] - b[fin]).max(initial=0.0)
        if self.fp16:
            if k == "hidden":
                self.fp16_hidden.append(numpy.abs(dev - b))
            return self._fp16({"hidden": "hidden", "priors": "priors"}.get(k, "logits"), err, what)
        if k == "priors":
            budget = self.k * numpy.abs(a - b).max() + 2 * b.max() * self.logit_budget(ref, "policy_logits", i) + self.floor
        else:
            budget = self.logit_budget(ref, k, i)
        self._ratio(err, budget, what)

    def scalar(self, what, dev, ref, k, i):
        a, b = ref[k][0][i], ref[k][1][i]
        err = abs(float(dev) - b)
        if self.fp16:
            return self._fp16("scalar", err, what)
        budget = (self.k * abs(a - b) + 2 * ref[k + "_sens"][i] * self.logit_budget(ref, k + "_logits", i)
                  + self.floor * max(1.0, abs(b)))
        self._ratio(err, budget, what)

    def finish(self):
        if not self.fp16:
            print(f"[net sweep] {self.name}: worst error/budget {self.worst:.3f} ({self.where})")
            return
        q = float(numpy.quantile(numpy.concatenate(self.fp16_hidden), 0.999)) if self.fp16_hidden else 0.0
        print(f"[net sweep] {self.name}: fp16 largest errors " +
              ", ".join(f"{k} {e:.3e} ({w})" for k, (e, w) in self.fp16_max.items()) + f", hidden 99.9% {q:.3e}")
        b = self.fp16_bounds
        for kind, bound in (("logits", b["logits"]), ("priors", 2 * b["logits"]), ("hidden", b["hidden_max"]),
                            ("scalar", b["scalar"])):
            err, where = self.fp16_max[kind]
            assert err <= bound, f"{self.name} {where}: fp16 error {err:.3e} > {bound:.3e}"
        assert q <= b["hidden_q999"], f"{self.name}: fp16 hidden 99.9% quantile {q:.3e} > {b['hidden_q999']:.3e}"


def _engine(case, mode, max_games, N, monkeypatch, parts=None):
    from muzero_general_b200.engine import SearchEngine
    for k in ("MZ_NO_TC", "MZ_NO_FUSE", "MZ_PARTS", "MZ_FC_GENERIC", "MZ_SMALL_SEARCH"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("MZ_TC_MODE", mode or "x3")
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    if parts is not None:
        monkeypatch.setenv("MZ_PARTS", str(parts))
    cfg = make_config(case)
    spec = case_spec(case)
    w = edge_weights(spec, case.weights)
    eng = SearchEngine(cfg, max_games=max_games, num_simulations=N)
    eng.load_weights(w)
    return cfg, spec, w, eng


def _pools(spec, n, seed=0):
    rs = numpy.random.RandomState(seed)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    hidden = rs.random_sample((n, spec.hidden_elems)).astype(numpy.float32)
    actions = (numpy.arange(n) % spec.action_space).astype(numpy.int32)
    return obs, hidden, actions


def _kernel_counts(eng, fn):
    eng.kernel_timing(True)
    eng.kernel_times()
    l0 = eng.launch_count
    fn()
    counts = {k: c for k, (_, c) in eng.kernel_times().items()}
    counts["launches"] = eng.launch_count - l0
    eng.kernel_timing(False)
    return counts


def _check_inference_route(case, spec, mode, eng, obs, hidden, actions):
    n = min(33, len(obs))
    init = _kernel_counts(eng, lambda: eng.initial_inference(obs[:n]))
    rec = _kernel_counts(eng, lambda: eng.recurrent_inference(hidden[:n], actions[:n]))
    num = eng.numerics
    tower, small, conv = "conv_tower_tc_kernel", "small_tower_kernel", "conv3x3_kernel"
    print(f"[net sweep] {case.name} [{mode}] numerics: {num}; kernels init {init}, rec {rec}")
    r = case.route
    if r.startswith("fc"):
        assert all(rec[k] == 0 for k in (tower, small, conv, "heads_kernel")), rec
        return
    if r == "tc":
        if case.weights in ("large", "tiny_bn", "overflow") and "left after" in num:
            return          # the range guard moved the net to the fp32 CUDA-core towers (printed above)
        assert {"x3": "f32-grade nets", "fp16": "fp16 operands"}[mode] in num, num
        assert rec[tower] >= 1 and rec[small] == 0 and rec[conv] == 0, rec
        assert (init[tower] >= 1) == (spec.blocks > 0) and init[conv] == 1, init
        return
    if case.env.get("MZ_TC_WIDE") == "3":           # the towers on the 256-channel x3 route, the stem on the CUDA cores
        assert "256-channel towers on the tensor cores" in num and rec[tower] >= 1 and init[tower] >= 1, (num, init, rec)
    else:
        assert "f32 nets" in num, num
        assert rec[tower] == 0 and init[tower] == 0
    if r == "tc_heads_left":
        assert "head weights exceed shared memory" in num, num
    if r in ("small_tower", "small_search"):
        towers = 2 if spec.blocks else 1            # (stem +) blocks of the first tower, blocks of the prediction tower
        assert rec[small] == towers and rec[conv] == 0 and init[small] == towers and init[conv] == 0, (init, rec)
    if r == "per_layer":
        assert rec[small] == 0 and rec[conv] == 1 + 4 * spec.blocks, rec
    if r == "downsample":
        assert init[conv] >= 1 + 4 + 1 + 6 + 6, init       # the stem's 18 convs stay on the CUDA cores on every route
    if r in ("heads_big", "tc_heads_left"):
        # generic heads: rescale + (1x1 conv + FC layers + scalar) per head, against 1 launch of heads_kernel
        assert init["launches"] >= 2 + 2 * 3 + 2, init
    if r == "heads_wide":
        assert rec["heads_kernel"] == 2, rec


def _judge_mode(case, mode, numerics):
    """The tolerance rule's mode: the tower mode on the tensor-core route, x3 for a DownSample net whose towers took the
    256-channel tensor-core route, fp32 otherwise."""
    if case.route == "tc":
        return mode if "left after" not in numerics else None
    return "x3" if numerics.startswith("f32-grade") else None


def _modes(case):
    if case.route == "tc_heads_left":
        return ["x3", "fp16"]          # either mode keeps these nets off the tensor cores from mz_create on
    if case.route != "tc":
        return [None]
    return ["x3", "fp16"] if case.weights == "synthetic" else ["x3"]


@pytest.mark.parametrize("name,mode", [(c.name, m) for c in CASES for m in _modes(c)])
def test_inference_matches_fp64_oracle(name, mode, monkeypatch):
    case = BY_NAME[name]
    spec = case_spec(case)
    batches = case.batches or (TC_BATCHES if case.route == "tc" else BATCHES)
    maxn = max(batches)
    _, spec, w, eng = _engine(case, mode, maxn, 2, monkeypatch)
    obs, hidden, actions = _pools(spec, maxn)
    _check_inference_route(case, spec, mode, eng, obs, hidden, actions)
    A = spec.action_space
    need = sorted(set().union(*[_rows(n, A, 1) for n in batches]))
    ref = Ref(spec, w)
    ri = ref.initial(obs[need])
    rr = ref.recurrent(hidden[need], actions[need])
    at = {r: j for j, r in enumerate(need)}
    judge = Judge(f"{name} [{mode or 'default'}]", _judge_mode(case, mode, eng.numerics), name)
    for n in batches:
        d0 = eng.initial_inference(obs[:n])
        d1 = eng.recurrent_inference(hidden[:n], actions[:n])
        for r in _rows(n, A, 1):
            j = at[r]
            tag = f"n={n} row {r}"
            judge.vector(f"{tag} init hidden", d0["hidden"][r], ri, "hidden", j)
            judge.vector(f"{tag} init value logits", d0["value_logits"][r], ri, "value_logits", j)
            judge.vector(f"{tag} init policy logits", d0["policy_logits"][r], ri, "policy_logits", j)
            judge.scalar(f"{tag} init value", d0["value"][r], ri, "value", j)
            assert d0["reward"][r] == 0 and numpy.isneginf(d0["reward_logits"][r]).sum() == 2 * spec.support_size
            judge.vector(f"{tag} rec hidden", d1["hidden"][r], rr, "hidden", j)
            judge.vector(f"{tag} rec value logits", d1["value_logits"][r], rr, "value_logits", j)
            judge.vector(f"{tag} rec reward logits", d1["reward_logits"][r], rr, "reward_logits", j)
            judge.vector(f"{tag} rec policy logits", d1["policy_logits"][r], rr, "policy_logits", j)
            judge.scalar(f"{tag} rec value", d1["value"][r], rr, "value", j)
            judge.scalar(f"{tag} rec reward", d1["reward"][r], rr, "reward", j)
            if case.weights == "const":
                C, HW = spec.channels, int(numpy.prod(spec.hidden_hw))
                for d in (d0, d1):
                    assert (d["hidden"][r].reshape(C, HW)[5] == 0).all(), "constant channel must rescale to exactly 0"
    judge.finish()
    eng.close()


# (case, tower mode, graph partitions); the small search runs without a trace (a traced search takes the step-wise
# pipeline), as does the partitioned replay (a traced search is never replayed)
SEARCH_RUNS = [("pl_9x9_c32", None, None), ("pl_c96_6x7", None, None), ("st_c32_6x7", None, None), ("ss_5x6_a4", None, None),
               ("ss_7x3_a12", None, None), ("tc_6x7", "x3", 1), ("tc_6x7", "x3", 2), ("tc_6x7", "fp16", 1), ("tc_6x7_b6", "x3", 2),
               ("tc_6x7_s300", "fp16", 1), ("tc_6x7_bigheads", "x3", 1), ("fc_cartpole", None, None),
               ("fc_cartpole_s20", None, None), ("fc_e5_a3", None, None), ("fc_a40", None, None),
               ("ds_breakout_96x96", None, None), ("ds_atari_96x96", None, None), ("ds_atari_96x96_wide", None, None)]
assert {r[0] for r in SEARCH_RUNS} == set(SEARCH_CASES)


@pytest.mark.parametrize("name,mode,parts", SEARCH_RUNS)
def test_search_network_outputs_match_fp64_oracle(name, mode, parts, monkeypatch):
    """The network numbers a search consumed, recomputed by the fp64 oracle from the device's own parent states (so
    errors do not compound): root hidden state, predicted value and priors against initial_inference(obs); for sampled
    expansions e, the hidden state, the reward of the edge into e, the priors of e's children and, where e was visited
    once, its value sum (exported tree), and with a trace the value / reward / priors of simulation e - 1, against
    recurrent_inference(hidden[parent(e)], action(e)).  The route is asserted on the very search whose outputs are
    checked (kernel timing only disables graph replay), except for the partitioned replay, which is replayed after an
    equal timed search."""
    case = BY_NAME[name]
    tc = case.route in ("tc", "tc_heads_left")
    n, N = (300, 12) if tc else (40, 12)
    _, spec, w, eng = _engine(case, mode, n, N, monkeypatch, parts)
    A = spec.action_space
    obs, _, _ = _pools(spec, n, seed=3)
    traced = parts != 2 and case.route != "small_search"
    kw = dict(obs=obs, add_exploration_noise=False, keep_tree=True, trace=traced)
    timed = []
    counts = _kernel_counts(eng, lambda: timed.append(eng.search(**kw)))
    print(f"[net sweep] search {name} [{mode}, parts {parts}] {eng.numerics}; kernels {counts}")
    r = case.route
    if r == "small_search":
        assert counts["small_search_kernel"] == 1 and counts["tree_step_kernel"] <= 1, counts    # (+ the root's step)
    elif r == "tc":
        assert counts["conv_tower_tc_kernel"] >= N and counts["small_search_kernel"] == 0, counts
    elif r == "tc_heads_left":
        assert "head weights exceed shared memory" in eng.numerics and counts["conv_tower_tc_kernel"] == 0, counts
    elif r == "small_tower":
        assert counts["small_tower_kernel"] >= N and counts["small_search_kernel"] == 0, counts
    elif r == "per_layer":
        assert counts["conv3x3_kernel"] >= N * (1 + 2 * spec.blocks), counts
    elif r in ("fc_fixed", "fc_generic"):
        assert counts["tree_step_kernel"] == 0, counts          # one launch of the fused FC search kernel
    elif r == "fc_stepwise":
        assert counts["tree_step_kernel"] >= N and counts["other"] >= N, counts      # tree steps + FC inference
    elif r == "downsample":
        assert counts["conv3x3_kernel"] >= 18, counts                               # the root's DownSample stem
    if parts == 2:
        for _ in range(3):          # eager, capture, replay of the partitioned graph
            out = eng.search(**kw)
        assert eng.graph_partitions == parts
    else:
        out = timed[0]
    ref = Ref(spec, w)
    judge = Judge(f"search {name} [{mode or 'default'}, parts {parts}]", _judge_mode(case, mode, eng.numerics), name)
    games = sorted({0, n // 2 - 1, n // 2, n - 1})
    ri = ref.initial(obs[games])
    for j, g in enumerate(games):
        tree = eng.export_tree(g, with_hidden=True)
        assert tree["n_expansions"] == N + 1
        judge.vector(f"game {g} root hidden", tree["hidden"][0], ri, "hidden", j)
        judge.scalar(f"game {g} root value", out.root_predicted_value[g], ri, "value", j)
        judge.vector(f"game {g} root priors", out.root_priors[g], ri, "priors", j)
        slot_of = {int(e): s for s, e in enumerate(tree["child_expansion"]) if e >= 0}
        exps = [1, 2, N // 2, N]
        parents = [slot_of[e] // A for e in exps]
        acts = [slot_of[e] % A for e in exps]
        rr = ref.recurrent(tree["hidden"][parents], acts)
        for k, e in enumerate(exps):
            tag = f"game {g} expansion {e}"
            s = slot_of[e]
            judge.vector(f"{tag} hidden", tree["hidden"][e], rr, "hidden", k)
            judge.scalar(f"{tag} edge reward", tree["child_reward"][s], rr, "reward", k)
            judge.vector(f"{tag} child priors", tree["child_prior"][e * A:(e + 1) * A], rr, "priors", k)
            if tree["child_visit"][s] == 1:          # a leaf backs its own value up with the sign of its player: +value
                judge.scalar(f"{tag} value sum", tree["child_value_sum"][s], rr, "value", k)
            if traced:
                tr = out.trace
                judge.scalar(f"{tag} traced value", tr["value"][g, e - 1], rr, "value", k)
                judge.scalar(f"{tag} traced reward", tr["reward"][g, e - 1], rr, "reward", k)
                judge.vector(f"{tag} traced priors", tr["priors"][g, e - 1], rr, "priors", k)
        assert tree["child_visit"][slot_of[N]] == 1           # the last expansion is a leaf: its value was checked
    judge.finish()
    eng.close()


def test_heads_beyond_shared_memory_keep_a_board_net_off_the_tensor_cores(monkeypatch):
    """The route of a 64-channel board net whose heads do not fit in shared memory is decided at mz_create, before any
    weights, in both tower modes: the hidden-state pool is then sized for the dense layout the CUDA-core route stores."""
    from muzero_general_b200.engine import SearchEngine
    for name in ("tc_6x7_s300", "tc_6x7_bigheads", "tc_6x7"):
        for mode in ("x3", "fp16"):
            monkeypatch.setenv("MZ_TC_MODE", mode)
            eng = SearchEngine(make_config(BY_NAME[name]), max_games=4, num_simulations=2)
            off = "head weights exceed shared memory" in eng.numerics
            assert off == (name != "tc_6x7"), (name, mode, eng.numerics)
            eng.close()
