// The reference's "lighter" representation stem, DownsampleCNN (models.py:278-297), fp32 on the CUDA cores:
// conv1 in -> mid = (in + C) / 2, k x k with k = 2 ceil(H / 16) (square), stride 4, padding 2, bias, ReLU, MaxPool(3, 2);
// conv2 mid -> C, 5 x 5, padding 2, bias, ReLU, MaxPool(3, 2); AdaptiveAvgPool to ceil(H / 16) x ceil(W / 16).
// Two launches of one kernel (cnn_stem.cu), the second with the average pool as its epilogue.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

namespace mz {

constexpr int kCnnStemThreads = 256;
constexpr int kCnnPlanLen = 36;           // int64 slots of a plan as mz_debug_cnn_stem_plan reports it

// Launch plan of one stage: conv (k, stride, pad 2) of n boards of cin x H x W -> cout x Ho x Wo, then MaxPool(3, 2) to
// Hp x Wp (and, for the second stage, the adaptive average to the hidden board).  A CTA owns `boards` boards, a tile of
// `co_tile` output channels and a band of `band` pooled rows; each thread owns 4 output channels of up to `items`
// conv pixels, whose partial sums stay in registers while the input channels are staged `cin_chunk` at a time.
struct CnnStagePlan {
    int cin, cout, H, W, k, stride, Ho, Wo, Hp, Wp;
    int co_tile, band, bands, boards, cin_chunk, items, threads;
    dim3 grid;                    // (board groups, channel tiles, bands)
    size_t smem;                  // dynamic shared memory bytes
};
struct CnnStemPlan {
    int h, w, mid;                // hidden board and conv1's output channels
    CnnStagePlan s[2];
};

// The plan of both stages for n boards of `in` planes of H x W and C channels on sm_count SMs (host only); false with
// the reason in *err - naming the stage that fails - for every geometry the reference's module cannot run.
bool cnn_stem_plan(int n, int in, int C, int H, int W, int sm_count, CnnStemPlan* p, std::string* err);
// plan -> the kCnnPlanLen values of mz_debug_cnn_stem_plan
void cnn_stem_plan_export(const CnnStemPlan& p, int64_t* out);

// Offsets (floats) of the stem's weights in a conv blob: conv weights [cin][k][k][cout], biases [cout]
struct CnnStemWeights { size_t w1, b1, w2, b2; };
// appends features.{0,3}.{weight, bias} (torch layout [cout][cin][k][k]) to the blob, each part 16-byte aligned
CnnStemWeights cnn_stem_pack(const float* w1, const float* b1, const float* w2, const float* b2, int in, int mid, int C, int k,
                             std::vector<float>& blob);

// stage 1: x [n][in][H][W] -> pooled [n][mid][Hp1][Wp1]; stage 2: -> out [n][C][h][w].  No host synchronisation.
cudaError_t cnn_stem_launch(const CnnStemPlan& p, const float* blob, const CnnStemWeights& w, const float* x, float* pooled,
                            float* out, int n, cudaStream_t stream);

// the stem alone on host NCHW data through cnn_stem_launch, the output filled with NaN first (mz_debug_cnn_stem)
int cnn_stem_debug(int n, int in, int C, int H, int W, const float* x, const float* w1, const float* b1, const float* w2,
                   const float* b2, float* out, int64_t* plan, int sm_count, std::string* err);

}  // namespace mz
