"""The fully-connected networks (csrc/fc_net.cuh) against plain references, case by case over tests/fccases.py, through
mz_debug_fc_net: fc_inference_kernel<G> as initial, recurrent and pool inference, and the fused search's two network calls
(its root evaluation and one simulation's recurrent inference, fc_search.cu fc_root_inference / fc_sim_inference run by a
debug kernel in the search's shared-memory layout, every game's region NaN bytes before the first layer).  Every output
starts as NaN bytes; every run asserts its plan.  Each stage is compared with fp64 of the device's own input to that stage,
which keeps the rescale's 1 / scale amplification out of the bounds.

  * exact: small integer weights, biases and inputs (partial sums below 2^24, pre-activations >= 0 or <= -104 so ELU is
    exact), the rescale pinned to a dyadic scale by two constant rows -M and +M of the last representation / dynamics layer:
    raw state, rescaled state and every exported logit EQUAL fp64, on every case, route and G
  * budget: standard-normal inputs, weights and biases, all scaled by gains 1, 1e-4 and 300; per Linear |W| d_in + gamma_{in+2} (|b| + |W| |x| + |Wx|),
    per ELU + 5u; the rescale bit for bit against a float32 restatement of the device's raw state (also constant states and
    states spanning ~1e-6, the 1e-5 rule); priors inside a first-order budget of the fp64 softmax of the device's logits;
    value and reward scalars by test_heads_gpu.check_scalar_budget on the device's logits; fc_inference_kernel's rescaled
    state, whose raw state is not exported, within the raw state's bound carried through the rescale
  * bit identity where the code claims it: the unrolled CartPole network equals the descriptors walk (many random weight
    sets, G 16 and 32), the heads side by side equal the heads one after the other, recurrent inference equals the search's
    simulation (and initial inference its root), each batch member equals its batch of one across grid-stride passes, pool
    inference equals recurrent inference on the gathered parents and writes only its slot
  * shared memory: fc_inference_kernel shrinks its CTA to fit (G = 4 with support 300, a net whose blob and one group's
    scratch fill the limit exactly); a net 16 bytes beyond is refused by mz_load_weights, and a new handle of the net at
    the limit loads it and serves it

Mutants of fc_net.cuh / fc_infer.cu / fc_search.cu, each built into the library and run against this file on an H100 80GB
HBM3 (396 tests; failing tests by test function):
  linear_layer not zeroing y[out..round4(out))          143: exact 99, budget 30, search call 9, others 5
  the generic one-hot row read as Wx[row + o]           199: exact 145, budget 49, fixed == walk 2, search call 2, smem 1
  the fixed path's one-hot row read as Wx[o A + action]  14: exact 4, budget 6, fixed == walk 2, search call 2
  the reward head fed the rescaled state (fused, fixed) 106: exact 38, budget 40, search call 14, side by side 12, fixed 2
  the < 1e-5 rule dropped (both rescales)                 2: constant / tiny-span rescale 2
  mlp_forward_multi reading in4[0] for every head        24: exact 9, budget 9, side by side 3, search call 3
  the fixed path's value and reward shuffles swapped      4: fixed == walk 2, search call 2
  pool inference writing slot gather_parent[g]            4: pool 3 (not pool_stride 1, where the slots coincide), the
                                                             G = 4 search (step-wise, pool calls) 1
"""
import zlib

import numpy
import pytest

from fccases import BY_NAME, CASES, INFER_ROUTES, SEARCH_ROUTES, SMEM_CAP, edge_case, groups_per_warp, one_pass, runs
import test_heads_gpu
from test_heads_gpu import check_scalar_budget, gamma

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ELU = 5.0
F32 = numpy.float32
WORST = {}


@pytest.fixture(scope="module")
def eng():
    from muzero_general_b200 import engine
    return engine


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def report(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))


def teardown_module(module):
    if WORST:
        print("\nworst measured error / bound:", {k: "%.3g" % v for k, v in sorted(WORST.items())})


# ---------------------------------------------------------------------------------------------------- references
def rescale_ref(raw):
    """models.py:138-145 in float32 (fc_net.cuh::rescale_unit_range): per-sample min-max, 1e-5 added to a scale < 1e-5."""
    raw = numpy.asarray(raw, F32)
    lo, hi = raw.min(1, keepdims=True), raw.max(1, keepdims=True)
    sc = hi - lo
    sc[sc < F32(1e-5)] += F32(1e-5)
    return (raw - lo) / sc


def mlp64(x, layers, d_in=0.0, action=None):
    """fp64 Linear / ELU stack of x [n, in] (layers: (W [out, in], b), the first layer's last A columns the one-hot rows
    when ``action`` is given) and the bound on the device's error given an error d_in on x."""
    h = numpy.asarray(x, numpy.float64)
    d = numpy.zeros_like(h) + d_in
    for l, (w, b) in enumerate(layers):
        w, b = numpy.asarray(w, numpy.float64), numpy.asarray(b, numpy.float64)
        dense = h.shape[1]
        wd = w[:, :dense]
        pre = h @ wd.T + b
        extra = numpy.zeros_like(pre)
        if l == 0 and action is not None:
            extra = w[:, dense + numpy.asarray(action)].T
            pre = pre + extra
        mag = numpy.abs(b) + (numpy.abs(h) + d) @ numpy.abs(wd).T + numpy.abs(extra)
        d = d @ numpy.abs(wd).T + gamma(dense + 2) * mag
        if l < len(layers) - 1:
            h = numpy.where(pre > 0, pre, numpy.expm1(numpy.minimum(pre, 0.0)))
            d = d + C_ELU * U
        else:
            h = pre
    return h, d


def softmax64(z):
    z = numpy.asarray(z, numpy.float64)
    e = numpy.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def check_prior(prior, z, dz, key):
    """prior vs the fp64 softmax of logits z known to within dz: expf's 2 ulp and the difference's rounding per entry, the
    sum's gamma_A, the division's u, and the logits' error to first order."""
    p = softmax64(z)
    A = z.shape[1]
    m = z.max(1, keepdims=True)
    dmax = numpy.max(dz, 1, keepdims=True) if numpy.ndim(dz) else dz
    bound = p * ((numpy.abs(z - m) + 6) * U + gamma(A) + numpy.expm1(4 * dmax)) + 2.0 ** -140
    err = numpy.abs(prior.astype(numpy.float64) - p)
    assert (err <= bound).all(), (key, float((err / bound).max()))
    report(key + " prior", (err / bound).max())


class _S:
    def __init__(self, S):
        self.S, self.name = S, "S%d" % S


def check_scalar(S, logits, scalar, key):
    check_scalar_budget(_S(S), {"logits": [logits], "scalar": numpy.asarray([scalar])}, key)
    report(key + " scalar", test_heads_gpu.WORST[key + " scalar"])


# ---------------------------------------------------------------------------------------------------- operands
def layers_of(case, weights):
    return {prefix: [(weights[f"{prefix}.{2 * l}.weight"], weights[f"{prefix}.{2 * l}.bias"]) for l in range(len(w) - 1)]
            for prefix, w in case.mlps()}


REP, DYN, REW, VAL, POL = ("representation_network.module", "dynamics_encoded_state_network.module",
                           "dynamics_reward_network.module", "prediction_value_network.module",
                           "prediction_policy_network.module")


def normal_weights(case, rs, gain=1.0):
    """Standard-normal weights (scaled by 1 / sqrt(fan-in)) and biases, every one times ``gain``: at gain 300 the logits
    spread over many orders of magnitude (expf underflows in the softmax and support_to_scalar), at 1e-4 they nearly
    cancel."""
    w = {}
    for prefix, widths in case.mlps():
        for l in range(len(widths) - 1):
            w[f"{prefix}.{2 * l}.weight"] = (rs.randn(widths[l + 1], widths[l]) / numpy.sqrt(widths[l]) * gain).astype(F32)
            w[f"{prefix}.{2 * l}.bias"] = (rs.randn(widths[l + 1]) * gain).astype(F32)
    return w


def int_weights(case, rs):
    w = {}
    for prefix, widths in case.mlps():
        for l in range(len(widths) - 1):
            dens = min(1.0, 8.0 / widths[l])
            w[f"{prefix}.{2 * l}.weight"] = (rs.randint(-1, 2, (widths[l + 1], widths[l])) *
                                             (rs.rand(widths[l + 1], widths[l]) < dens)).astype(F32)
            w[f"{prefix}.{2 * l}.bias"] = rs.randint(-3, 4, widths[l + 1]).astype(F32)
    return w


def fix_biases(layers, x, rs, action=None):
    """Hidden biases keeping every hidden unit >= 0 for every sample or <= -104 for every sample (ELU exact)."""
    h = numpy.asarray(x, numpy.float64)
    for l, (w, b) in enumerate(layers[:-1]):
        z = h @ w[:, :h.shape[1]].astype(numpy.float64).T
        if l == 0 and action is not None:
            z = z + w[:, h.shape[1] + action].T
        up = rs.rand(len(b)) < 0.6
        # integer biases: exact in float32 whatever the (dyadic) inputs
        b[:] = numpy.where(up, numpy.ceil(-z.min(0)) + rs.randint(0, 3, len(b)),
                           numpy.floor(-z.max(0)) - 104 - rs.randint(0, 3, len(b)))
        pre = z + b
        assert ((pre >= 0).all(0) | (pre <= -104).all(0)).all()
        h = numpy.where(pre >= 0, pre, -1.0)             # ELU(0) = expf(0) - 1 = 0
    return h


def pin(layers, x, action):
    """Rows 0 and 1 of the last layer: zero weights, biases -M and +M with M a power of two above every other row."""
    w, b = layers[-1]
    if w.shape[0] < 2:
        return None
    w[:2] = 0
    raw, _ = mlp64(x, layers, action=action)
    M = 2.0 ** numpy.ceil(numpy.log2(numpy.abs(raw).max() + 2))
    b[0], b[1] = -M, M
    return M


def exact_operands(case, rs, n, route):
    w = int_weights(case, rs)
    L = layers_of(case, w)
    A, E = case.A, case.E
    action = rs.randint(0, A, n)
    if route in ("infer_initial", "search_root"):
        x = rs.randint(-3, 4, (n, case.obs)).astype(F32)
        fix_biases(L[REP], x, rs)
        pin(L[REP], x, None)
        raw, _ = mlp64(x, L[REP])
    else:
        x = rs.randint(-3, 4, (n, E)).astype(F32)
        fix_biases(L[DYN], x, rs, action)
        pin(L[DYN], x, action)
        raw, _ = mlp64(x, L[DYN], action=action)
    hid = rescale_ref(raw.astype(F32))
    for prefix, inp in ((REW, raw), (VAL, hid), (POL, hid)):
        fix_biases(L[prefix], inp, rs)
    return w, x, action


def run(eng, case, G, route, w, x, action=None, n_check=None, **kw):
    n = x.shape[0]
    parents = kw.pop("parents", None)
    if route == "infer_pool" and parents is None:
        parents = numpy.zeros(n, numpy.int32)
    out = eng.debug_fc_net(case.spec(), w, G, route, x, actions=action, parents=parents, **kw)
    want, why = eng.debug_fc_net_plan(case.spec(), G, route, n, force_split=kw.get("force_split", False),
                                      sm_count=n_check or 132, smem_cap=SMEM_CAP)
    if n_check:
        assert out["plan"] == want, (case.name, G, route, out["plan"], want)
    return out


def nan(a):
    return (numpy.asarray(a, F32).view(numpy.uint32) == 0xFFFFFFFF).all()


def exported(case, route, path):
    """Which logits the route writes."""
    if route in INFER_ROUTES:
        return {"policy_logits", "value_logits", "reward_logits"}
    if path == "fixed" and route == "search_sim":        # the search's root always walks the descriptors
        return set()
    return {"policy_logits", "value_logits"} | ({"reward_logits"} if route == "search_sim" else set())


def check_nan_contract(case, route, out):
    path = out["plan"]["path"]
    for k in ("policy_logits", "value_logits", "reward_logits"):
        if k not in exported(case, route, path):
            assert nan(out[k]), (case.name, route, k, "written")
    if route in INFER_ROUTES:
        assert nan(out["raw"]) and nan(out["prior"])
    if route == "search_root":
        assert nan(out["reward"])


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("name,G,route", runs())
def test_exact_on_integer_operands(eng, sm_count, name, G, route):
    case = BY_NAME[name]
    rs = numpy.random.RandomState(zlib.crc32(f"{name} {G} {route}".encode()))
    n = groups_per_warp(G) + 1 + 4
    w, x, action = exact_operands(case, rs, n, route)
    L = layers_of(case, w)
    out = run(eng, case, G, route, w, x, action if route in ("infer_recurrent", "infer_pool", "search_sim") else None,
              n_check=sm_count)
    check_nan_contract(case, route, out)
    if route in ("infer_initial", "search_root"):
        raw, _ = mlp64(x, L[REP])
    else:
        raw, _ = mlp64(x, L[DYN], action=action)
    hid = rescale_ref(raw.astype(F32))
    if route in SEARCH_ROUTES:
        assert numpy.array_equal(out["raw"].astype(numpy.float64), raw), (name, G, route, "raw")
    assert numpy.array_equal(out["hidden"].view(numpy.uint32), hid.view(numpy.uint32)), (name, G, route, "hidden")
    want = {"policy_logits": mlp64(hid, L[POL])[0], "value_logits": mlp64(hid, L[VAL])[0], "reward_logits": mlp64(raw, L[REW])[0]}
    if route == "infer_initial":
        want["reward_logits"] = numpy.where(numpy.arange(case.F) == case.S, 0.0, -numpy.inf)[None].repeat(n, 0)
    for k in exported(case, route, out["plan"]["path"]):
        assert numpy.array_equal(out[k].astype(numpy.float64), want[k]), (name, G, route, k)
    if route == "infer_pool":
        assert numpy.array_equal(out["pool"][:, 0].view(numpy.uint32), hid.view(numpy.uint32))


def budget_operands(case, rs, n, gain, route):
    w = normal_weights(case, rs, gain)
    if route in ("infer_initial", "search_root"):
        x = (rs.randn(n, case.obs) * gain).astype(F32)
    else:
        x = (rs.randn(n, case.E) * gain).astype(F32)
    return w, x, rs.randint(0, case.A, n).astype(numpy.int32)


def check_rescale_bound(case, hid, raw, draw, key):
    """fc_inference_kernel's rescaled state (its raw state is not exported) against the rescale of the fp64 raw state, which
    the device's raw state matches within draw: with dm the sample's largest raw error, the extrema move by dm and the scale
    by 2 dm, so |hid - (x - lo) / sc| <= (|x - lo| + draw + dm) / (sc - 2 dm) (1 + 8u) - |x - lo| / sc (five roundings, with
    1e-5 in float32).  Samples whose scale is within its error of the 1e-5 threshold are left to the exact test.  A one-element
    state is its own minimum: it rescales to exactly 0."""
    if case.E == 1:
        assert (hid == 0).all(), (case.name, key, "hidden")
        return
    lo, hi = raw.min(1, keepdims=True), raw.max(1, keepdims=True)
    sc = hi - lo
    dm = draw.max(1, keepdims=True)
    sure = (numpy.abs(sc - 1e-5) > 2 * dm + 4 * U * sc).ravel()
    sc = numpy.where(sc < 1e-5, sc + 1e-5, sc)
    sure &= (sc > 4 * dm).ravel()
    num = raw - lo
    bound = (num + draw + dm) / (sc - 2 * dm) * (1 + 8 * U) - num / sc + 2.0 ** -140
    err = numpy.abs(hid.astype(numpy.float64) - num / sc)
    assert (err[sure] <= bound[sure]).all(), (case.name, key, "hidden", float((err[sure] / bound[sure]).max()))
    assert sure.sum() >= len(sure) // 2, (case.name, key, "too few samples away from the 1e-5 threshold")
    report(key + " inference state", (err[sure] / bound[sure]).max())


def check_budget(case, route, w, x, action, out, key):
    L = layers_of(case, w)
    recurrent = route not in ("infer_initial", "search_root")
    raw, draw = mlp64(x, L[DYN], action=action) if recurrent else mlp64(x, L[REP])
    if route in SEARCH_ROUTES:
        err = numpy.abs(out["raw"] - raw)
        assert (err <= draw).all(), (case.name, key, "raw", float((err / draw).max()))
        report(key + " raw", (err / numpy.maximum(draw, 1e-300)).max())
        assert numpy.array_equal(out["hidden"].view(numpy.uint32), rescale_ref(out["raw"]).view(numpy.uint32)), (case.name, key)
        raw, draw = out["raw"].astype(numpy.float64), 0.0
    else:
        check_rescale_bound(case, out["hidden"], raw, draw, key)
    hid = out["hidden"]
    path = out["plan"]["path"]
    heads = {"policy_logits": mlp64(hid, L[POL]), "value_logits": mlp64(hid, L[VAL]), "reward_logits": mlp64(raw, L[REW], draw)}
    for k in exported(case, route, path):
        if k == "reward_logits" and route == "infer_initial":
            continue
        want, d = heads[k]
        err = numpy.abs(out[k] - want)
        assert (err <= d).all(), (case.name, key, k, float((err / d).max()))
        report(key + " logits", (err / numpy.maximum(d, 1e-300)).max())
    if route in SEARCH_ROUTES:
        if "policy_logits" in exported(case, route, path):
            check_prior(out["prior"], out["policy_logits"], 0.0, key)
        else:
            check_prior(out["prior"], *heads["policy_logits"], key)
    if "value_logits" in exported(case, route, path):
        check_scalar(case.S, out["value_logits"], out["value"], key + " value")
    if route != "search_root" and "reward_logits" in exported(case, route, path) and route != "infer_initial":
        check_scalar(case.S, out["reward_logits"], out["reward"], key + " reward")


@pytest.mark.parametrize("gain", [1.0, 1e-4, 300.0])
@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_inside_fp64_budget(eng, name, gain):
    case = BY_NAME[name]
    for G in case.groups:
        for route in INFER_ROUTES + SEARCH_ROUTES:
            if route in SEARCH_ROUTES and case.A > G:
                continue
            rs = numpy.random.RandomState(zlib.crc32(f"{name} {gain} {G} {route}".encode()))
            w, x, action = budget_operands(case, rs, 45, gain, route)
            out = run(eng, case, G, route, w, x, action)
            check_nan_contract(case, route, out)
            check_budget(case, route, w, x, action, out, "gain %g" % gain)


@pytest.mark.parametrize("route", ["search_root", "search_sim"])
def test_rescale_of_constant_and_tiny_span_states(eng, route):
    """The last representation / dynamics layer's weights zeroed: every sample's raw state is its biases - constant, or
    spanning ~1e-6 (scale < 1e-5 gets 1e-5 added): the rescaled state equals the float32 restatement bit for bit."""
    for name in ("cartpole", "e5_a7_split", "e36_a17_obs301"):
        case = BY_NAME[name]
        for G in case.search_groups():
            for spread in (0.0, 1e-6, 3e-5):
                rs = numpy.random.RandomState(7)
                w = normal_weights(case, rs)
                prefix, n_l = (REP, len(case.rep)) if route == "search_root" else (DYN, len(case.dyn))
                w[f"{prefix}.{2 * n_l}.weight"][:] = 0
                w[f"{prefix}.{2 * n_l}.bias"][:] = F32(0.37) * (1 + spread * rs.rand(case.E)).astype(F32)
                x = rs.randn(9, case.obs if route == "search_root" else case.E).astype(F32)
                out = run(eng, case, G, route, w, x, rs.randint(0, case.A, 9))
                assert numpy.array_equal(out["hidden"].view(numpy.uint32), rescale_ref(out["raw"]).view(numpy.uint32))
                assert numpy.array_equal(out["raw"], numpy.broadcast_to(w[f"{prefix}.{2 * n_l}.bias"], out["raw"].shape))


SEARCH_KEYS = ("raw", "hidden", "prior", "value", "reward")


@pytest.mark.parametrize("G", [16, 32])
def test_fixed_cartpole_network_equals_the_descriptors_walk(eng, G):
    """fc_recurrent_fixed against the generic walk (forced split: the heads one after the other) on 40 random CartPole-shaped
    weight sets: next, rescaled state, prior, value and reward bit for bit."""
    case = BY_NAME["cartpole"]
    for seed in range(40):
        rs = numpy.random.RandomState(seed)
        gain = (1.0, 1e-4, 300.0)[seed % 3]
        w, x, action = budget_operands(case, rs, 37, gain, "search_sim")
        fixed = run(eng, case, G, "search_sim", w, x, action)
        split = run(eng, case, G, "search_sim", w, x, action, force_split=True)
        assert fixed["plan"]["path"] == "fixed" and split["plan"]["path"] == "split"
        for k in SEARCH_KEYS:
            assert numpy.array_equal(fixed[k].view(numpy.uint32), split[k].view(numpy.uint32)), (G, seed, k)


@pytest.mark.parametrize("name", [c.name for c in CASES if c.path_wide == "fused" and c.search_groups()])
def test_heads_side_by_side_equal_one_after_the_other(eng, name):
    case = BY_NAME[name]
    for G in case.search_groups():
        rs = numpy.random.RandomState(3)
        w, x, action = budget_operands(case, rs, 37, 1.0, "search_sim")
        fused = run(eng, case, G, "search_sim", w, x, action)
        split = run(eng, case, G, "search_sim", w, x, action, force_split=True)
        assert fused["plan"]["path"] == "fused" and split["plan"]["path"] == "split"
        for k in SEARCH_KEYS + ("policy_logits", "value_logits", "reward_logits"):
            assert numpy.array_equal(fused[k].view(numpy.uint32), split[k].view(numpy.uint32)), (name, G, k)


@pytest.mark.parametrize("name", [c.name for c in CASES if c.search_groups()])
def test_inference_equals_the_search_call(eng, name):
    """infer_recurrent equals search_sim (and infer_initial search_root) on the rescaled state, the logits the search exports
    and the scalars."""
    case = BY_NAME[name]
    for G in case.search_groups():
        for inf, srch in (("infer_recurrent", "search_sim"), ("infer_initial", "search_root")):
            rs = numpy.random.RandomState(5)
            w, x, action = budget_operands(case, rs, 37, 1.0, srch)
            a = run(eng, case, G, inf, w, x, action)
            b = run(eng, case, G, srch, w, x, action)
            keys = ["hidden", "value"] + (["reward"] if srch == "search_sim" else [])
            keys += sorted(exported(case, srch, b["plan"]["path"]))
            for k in keys:
                assert numpy.array_equal(a[k].view(numpy.uint32), b[k].view(numpy.uint32)), (name, G, inf, k)


@pytest.mark.parametrize("name,G", [("cartpole", 4), ("cartpole", 16), ("e3_a3_unequal_widths", 8),
                                    ("e36_a17_obs301", 32), ("g4_s300_flat", 4)])
def test_batch_members_equal_a_batch_of_one(eng, sm_count, name, G):
    """A batch of one grid pass + 1 (several passes when the CTA shrinks): every member, also the groups re-evaluating the
    last sample, stores what a batch of one stores, on every route."""
    case = BY_NAME[name]
    routes = INFER_ROUTES + (SEARCH_ROUTES if case.A <= G else ())
    for route in routes:
        plan, _ = eng.debug_fc_net_plan(case.spec(), G, route, 1, sm_count=sm_count)
        n = one_pass(G, sm_count, plan["threads"]) + 1 if route in INFER_ROUTES else 8 * sm_count * (32 // G) + 1
        rs = numpy.random.RandomState(9)
        w, x, action = budget_operands(case, rs, n, 1.0, route)
        big = run(eng, case, G, route, w, x, action, n_check=sm_count)
        assert big["plan"]["grid"] == 8 * sm_count
        for i in sorted({0, 1, groups_per_warp(G), n // 2, n - 2, n - 1}):
            one = run(eng, case, G, route, w, x[i:i + 1], action[i:i + 1])
            for k in ("hidden", "raw", "prior", "value", "reward", "policy_logits", "value_logits", "reward_logits"):
                assert numpy.array_equal(big[k][i].view(numpy.uint32), one[k][0].view(numpy.uint32)), (name, G, route, i, k)


@pytest.mark.parametrize("pool_stride,slots", [(1, (0, 0)), (3, (0, 2)), (3, (2, 0)), (3, (1, 1))])
def test_pool_inference_gathers_its_parents_and_writes_its_slot(eng, pool_stride, slots):
    for name in ("cartpole", "e5_a7_split", "e8_a256_infer"):
        case = BY_NAME[name]
        rs = numpy.random.RandomState(pool_stride)
        n = 37
        w, x, action = budget_operands(case, rs, n, 1.0, "infer_recurrent")
        parent_slot, out_slot = slots
        parents = numpy.full(n, parent_slot, numpy.int32)
        parents[::2] = (parent_slot + 1) % pool_stride if pool_stride > 1 else 0
        for G in case.groups:
            ref = run(eng, case, G, "infer_recurrent", w, x, action)
            pool = run(eng, case, G, "infer_pool", w, x, action, parents=parents, pool_stride=pool_stride, out_slot=out_slot)
            for k in ("hidden", "value", "reward", "policy_logits", "value_logits", "reward_logits"):
                assert numpy.array_equal(pool[k].view(numpy.uint32), ref[k].view(numpy.uint32)), (name, G, k)
            p = pool["pool"]
            assert numpy.array_equal(p[:, out_slot].view(numpy.uint32), ref["hidden"].view(numpy.uint32))
            for g in range(n):
                for s in range(pool_stride):
                    if s == out_slot:
                        continue
                    if s == parents[g]:
                        assert numpy.array_equal(p[g, s], x[g]), (name, G, g, "parent slot changed")
                    else:
                        assert nan(p[g, s]), (name, G, g, s, "another slot written")


# ---------------------------------------------------------------------------------------------------- shared memory
def test_inference_fits_its_cta_to_shared_memory(eng):
    """G = 4 with support 300 (128 threads would need 32 x 2420 floats of scratch) and a net whose blob and one group's
    scratch are exactly the limit: served, inside the budget."""
    for case, G in ((BY_NAME["g4_s300_flat"], 4), (edge_case(0), 32)):
        for route in INFER_ROUTES:
            rs = numpy.random.RandomState(1)
            w, x, action = budget_operands(case, rs, 300, 1.0, route)
            out = run(eng, case, G, route, w, x, action)
            assert out["plan"]["smem"] <= SMEM_CAP
            check_nan_contract(case, route, out)
            check_budget(case, route, w, x, action, out, "smem edge")
    assert eng.debug_fc_net_plan(edge_case(0).spec(), 32, "infer_initial", 1)[0]["smem"] == SMEM_CAP


def engine_for(case, monkeypatch, G):
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module("cartpole").MuZeroConfig()
    cfg.observation_shape = (1, 1, case.obs)
    cfg.action_space = list(range(case.A))
    cfg.encoding_size, cfg.support_size = case.E, case.S
    cfg.fc_representation_layers, cfg.fc_dynamics_layers = list(case.rep), list(case.dyn)
    cfg.fc_reward_layers, cfg.fc_value_layers, cfg.fc_policy_layers = list(case.rew), list(case.val), list(case.pol)
    monkeypatch.setenv("MZ_FC_GROUP", str(G))
    return SearchEngine(cfg, max_games=8, num_simulations=4)


def test_load_refuses_a_net_beyond_shared_memory_and_serves_the_next(eng, monkeypatch):
    """A net 16 bytes (one 4-float granule of the blob) beyond the limit is refused by mz_load_weights with both byte counts,
    not at its first call, and the refused handle stays consistent (it has no weights).  A handle's network shape is fixed
    when it is created, so a new handle, of the net at the limit, then loads it and serves it."""
    from muzero_general_b200._lib import MzError
    beyond, at = edge_case(16), edge_case(0)
    rs = numpy.random.RandomState(2)
    x = rs.randn(5, at.obs).astype(F32)
    e = engine_for(beyond, monkeypatch, 32)
    try:
        with pytest.raises(MzError) as info:
            e.load_weights(normal_weights(beyond, rs))
        assert str(SMEM_CAP + 16) in str(info.value) and str(SMEM_CAP) in str(info.value), str(info.value)
        with pytest.raises(MzError, match="weights not loaded"):
            e.initial_inference(x)
    finally:
        e.close()
    e = engine_for(at, monkeypatch, 32)
    try:
        w = normal_weights(at, rs)
        e.load_weights(w)
        got = e.initial_inference(x)
        want = run(eng, at, 32, "infer_initial", w, x)
        for k in ("value", "value_logits", "policy_logits"):
            assert numpy.array_equal(got[k].view(numpy.uint32), want[k].view(numpy.uint32)), k
    finally:
        e.close()


def test_g4_support_300_serves_inference_and_search(eng, monkeypatch):
    """With MZ_FC_GROUP=4 and support 300 every inference used to fail to launch (128 threads' scratch over the limit)."""
    case = BY_NAME["g4_s300_flat"]
    e = engine_for(case, monkeypatch, 4)
    try:
        rs = numpy.random.RandomState(4)
        w = normal_weights(case, rs)
        e.load_weights(w)
        x = rs.randn(6, case.obs).astype(F32)
        got = e.initial_inference(x)
        want = run(eng, case, 4, "infer_initial", w, x)
        assert numpy.array_equal(got["value"].view(numpy.uint32), want["value"].view(numpy.uint32))
        out = e.search(obs=x, legal_mask=numpy.ones((6, case.A), numpy.uint8))
        assert (out.visit_counts.sum(1) == 4).all()
    finally:
        e.close()
