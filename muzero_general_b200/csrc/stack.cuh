// The rule of a stacked network input (GameHistory.get_stacked_observations(t, s, A), self_play.py:304-315), shared by
// the self-play loop (stack_fill, selfplay.cu) and Reanalyse (reanalyse_stack_kernel, reanalyse.cu).
#pragma once
#include "common.cuh"

namespace mz {

// Element e of the stacked tail of position t's input, the s * (O + plane) floats after its own observation: block
// k = e / (O + plane) belongs to p = t - 1 - k and holds observation p (frame(p)[j] for j < O), then a plane of
// action_history[p + 1] / A (action(p) returns action_history[p + 1]); the whole block is zeros when p < 0.  The plane
// is the fp64 quotient rounded once to fp32, what the reference's float64 plane becomes after .float().
template <class Frame, class Action>
MZ_DEVINL float stack_tail_element(int e, int t, int O, int plane, int A, const Frame& frame, const Action& action) {
    const int block = O + plane;
    const int k = e / block, j = e - k * block, p = t - 1 - k;
    if (p < 0) return 0.0f;
    return j < O ? frame(p)[j] : __double2float_rn(__ddiv_rn((double)action(p), (double)A));
}

}  // namespace mz
