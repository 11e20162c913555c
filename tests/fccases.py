"""Case table of the fully-connected networks (csrc/fc_net.cuh, csrc/fc_infer.cu and the search's network calls in
csrc/fc_search.cu, reached through mz_debug_fc_net / mz_debug_fc_net_plan).  Importable without a GPU.

Each case is one network shape and the lane groups it runs at.  Every case runs the three fc_inference_kernel routes at
every G it lists; the search routes run where the search can (action_space <= G).  Together the cases reach:
  * fc_inference_kernel<G> for G = 4, 8, 16, 32, and the CTA sized down from 128 threads when the scratch does not fit
  * the search's paths: the unrolled CartPole network (fixed) at G 16 and 32, the descriptors walk with the heads side by
    side (fused) and one after the other (split) at G 4, 8, 16 and 32
  * near-misses of the fixed shape, one field off, which take the generic path (the representation network is not part of
    the fixed shape: a representation with no hidden layer stays fixed)
  * E in {1, 3, 5, 8, 32, 36, 64}, observations of 1 to 301 floats (odd sizes; 301 sets the widest vector), hidden lists
    [], [3], [16], [33], [3, 9], [128, 128], heads of equal depth and unequal widths, S in {0, 4, 10, 20, 300}, A in
    {1, 2, 3, 4, 7, 8, 17, 32} in the search and up to 256 on the inference routes
"""
from dataclasses import dataclass, replace
from typing import Tuple

SMS = (132, 114)                  # H100 SXM and PCIe
SMEM_CAP = 232448                 # H100's shared memory per block (opt-in)


@dataclass(frozen=True)
class FcCase:
    name: str
    obs: int
    E: int
    A: int
    S: int
    rep: Tuple[int, ...]
    dyn: Tuple[int, ...]
    rew: Tuple[int, ...]
    val: Tuple[int, ...]
    pol: Tuple[int, ...]
    groups: Tuple[int, ...] = (4, 8, 16, 32)
    # the search's path at G 16 / 32 ("fixed" only for the CartPole shape) and at G 4 / 8
    path_wide: str = "fused"
    path_narrow: str = "fused"

    @property
    def F(self):
        return 2 * self.S + 1

    def spec(self):
        from muzero_general_b200.netspec import FC, NetSpec
        return NetSpec(kind=FC, obs_shape=(self.obs, 1, 1), stacked=0, in_channels=self.obs, action_space=self.A,
                       support_size=self.S, encoding=self.E, fc_representation=list(self.rep), fc_dynamics=list(self.dyn),
                       fc_reward=list(self.rew), fc_value=list(self.val), fc_policy=list(self.pol))

    def search_groups(self):
        return tuple(G for G in self.groups if self.A <= G)

    def search_path(self, G):
        return self.path_wide if G >= 16 else self.path_narrow

    def mlps(self):
        """(state_dict prefix, widths) of the five MLPs, as netspec.weights_spec names them."""
        E, A, F = self.E, self.A, self.F
        return [("representation_network.module", [self.obs, *self.rep, E]),
                ("dynamics_encoded_state_network.module", [E + A, *self.dyn, E]),
                ("dynamics_reward_network.module", [E, *self.rew, F]),
                ("prediction_value_network.module", [E, *self.val, F]),
                ("prediction_policy_network.module", [E, *self.pol, A])]


H16 = (16,)
CASES = [
    # games/cartpole.py: the fixed path at G 16 / 32
    FcCase("cartpole", 4, 8, 2, 10, H16, H16, H16, H16, H16, path_wide="fixed"),
    FcCase("cartpole_rep_none", 4, 8, 2, 10, (), H16, H16, H16, H16, path_wide="fixed"),
    # near-misses: one field off
    FcCase("cartpole_rew_16_16", 4, 8, 2, 10, H16, H16, (16, 16), H16, H16, path_wide="split", path_narrow="split"),
    FcCase("cartpole_a3", 4, 8, 3, 10, H16, H16, H16, H16, H16),
    FcCase("cartpole_s20", 4, 8, 2, 20, H16, H16, H16, H16, H16),
    FcCase("cartpole_e12", 4, 12, 2, 10, H16, H16, H16, H16, H16),
    FcCase("cartpole_h20", 4, 8, 2, 10, H16, (20,), (20,), (20,), (20,)),
    # edges
    FcCase("e1_a1_s0", 1, 1, 1, 0, (), (), (), (), ()),
    FcCase("e1_a1_s4_hidden", 3, 1, 1, 4, (3,), (3,), (3,), (3,), (3,)),
    FcCase("e3_a3_unequal_widths", 7, 3, 3, 4, (3,), (3, 9), (33,), H16, (3,)),
    FcCase("e5_a7_split", 13, 5, 7, 4, (3, 9), (33,), (3, 9), H16, (), path_wide="split", path_narrow="split"),
    FcCase("e8_a4_s300", 9, 8, 4, 300, (33,), H16, (3,), (33,), H16, groups=(8, 16, 32)),
    FcCase("e36_a17_obs301", 301, 36, 17, 20, (33,), (128, 128), (33,), (33,), (33,), groups=(32,)),
    FcCase("e32_a8_flat", 5, 32, 8, 10, (), (), (), (), (), groups=(8, 16, 32)),
    FcCase("e64_a32_deep", 64, 64, 32, 10, (128, 128), (33,), (33,), (3, 9), (33,), groups=(4, 32),
           path_wide="split", path_narrow="split"),
    FcCase("e8_a8_wide_heads", 6, 8, 8, 10, (3,), (3,), (128, 128), (128, 128), (3, 9), groups=(8, 32)),
    FcCase("e3_a2_wide_policy", 2, 3, 2, 4, H16, H16, H16, H16, (128, 128), groups=(16,),
           path_wide="split"),
    # inference only (action_space > 32)
    FcCase("e8_a256_infer", 10, 8, 256, 10, H16, H16, H16, H16, (33,)),
    # fc_inference_kernel's scratch does not fit 128 threads: at G = 4 the CTA has 64 threads
    FcCase("g4_s300_flat", 4, 8, 2, 300, (), (), (), (), (), groups=(4,)),
]
BY_NAME = {c.name: c for c in CASES}

INFER_ROUTES = ("infer_initial", "infer_recurrent", "infer_pool")
SEARCH_ROUTES = ("search_root", "search_sim")


def runs(routes=INFER_ROUTES + SEARCH_ROUTES):
    """(case name, G, route) of every run of the table."""
    out = []
    for c in CASES:
        for G in c.groups:
            for r in routes:
                if r in SEARCH_ROUTES and G < c.A:
                    continue
                out.append((c.name, G, r))
    return out


def groups_per_warp(G):
    return 32 // G


def one_pass(G, sms, threads=128):
    """Samples of one grid-stride pass of fc_inference_kernel<G> (8 CTAs per SM)."""
    return 8 * sms * (threads // G)


def infer_smem(case, G, groups):
    """fc_inference_kernel's shared memory: the blob (rounded to 4 floats), then 4 maxw + 4 floats per group."""
    return ((blob_floats(case) + 3) & ~3) * 4 + groups * (4 * maxw(case) + 4) * 4


def maxw(case):
    w = max(case.E, case.F, case.A, case.obs)
    for _, widths in case.mlps():
        w = max(w, *widths[1:])
    return (w + 3) & ~3


def blob_floats(case):
    """Floats of the packed weight blob (abi.cu pack_mlp): per Linear the weights [ceil(in_dense / 4)][out][4] at a
    multiple of 4, the bias, and for the first dynamics layer the A one-hot rows."""
    n = 0
    for k, (_, widths) in enumerate(case.mlps()):
        for l in range(len(widths) - 1):
            extra = case.A if (k == 1 and l == 0) else 0
            n = (n + 3) & ~3
            n += ((widths[l] - extra + 3) // 4) * widths[l + 1] * 4 + widths[l + 1] + extra * widths[l + 1]
    return n


def edge_case(total_bytes_over):
    """A flat E = 1 net (G = 32, one group per warp) whose blob plus one group's scratch is SMEM_CAP + total_bytes_over."""
    base = replace(BY_NAME["e1_a1_s0"], groups=(32,))
    want = SMEM_CAP + total_bytes_over
    for S in range(40, 2000):
        lo, hi = 1, 20000                   # the bytes grow with the representation's hidden width h: bisect for it
        while lo < hi:
            mid = (lo + hi) // 2
            if infer_smem(replace(base, S=S, rep=(mid,)), 32, 1) < want:
                lo = mid + 1
            else:
                hi = mid
        c = replace(base, S=S, rep=(lo,), name=f"edge{total_bytes_over:+d}")
        if infer_smem(c, 32, 1) == want:
            return c
    raise AssertionError("no edge shape")
