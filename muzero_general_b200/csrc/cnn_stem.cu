// DownsampleCNN stem (cnn_stem.h): two launches of cnn_stage_kernel, fp32 on the CUDA cores.
//
// A CTA owns (boards, a tile of output channels, a band of pooled rows).  It computes the conv rows its pooled rows
// read - 2 * band + 1 of them, the 3/2 windows of neighbouring pooled rows share one - for all its boards into shared
// memory, then max-pools from there: the un-pooled conv output never goes to global memory.  The second stage holds
// the whole pooled plane of its channels, so it also computes the adaptive average bins and writes the hidden board.
//
// Arithmetic, per conv output: acc = 0; acc = fma(x, w, acc) over (ci, ky, kx) in that order (padding taps multiply a
// staged zero); then acc + bias; ReLU.  The max pool is exact.  Each average is the fp32 sum of its bin, rows then
// columns, divided once, correctly rounded (__fdiv_rn), by the bin's element count.
#include "cnn_stem.h"

#include <algorithm>

#include "../../include/mzb200.h"
#include "launch.h"

namespace mz {

namespace {

struct CnnStageArgs : CnnStagePlan {
    const float* in;          // [n][cin][H][W]
    float* out;               // [n][cout][Hp][Wp], or [n][cout][avg_h][avg_w] with the average epilogue
    const float* w;           // [cin][k][k][cout]
    const float* bias;        // [cout]
    int n, avg_h, avg_w;      // avg_h = 0: no average pool
};

template <int ITEMS>
__global__ void __launch_bounds__(kCnnStemThreads) cnn_stage_kernel(const __grid_constant__ CnnStageArgs a) {
    extern __shared__ __align__(16) float smem[];
    pdl_launch_dependents();
    const int CO = a.co_tile, cgs = CO / 4, lanes = blockDim.x / cgs;
    const int cg = threadIdx.x % cgs, lane = threadIdx.x / cgs;
    const int b0 = blockIdx.x * a.boards, nb = min(a.boards, a.n - b0);
    const int co0 = blockIdx.y * CO, cov = min(CO, a.cout - co0);
    const int p0 = blockIdx.z * a.band, npr = min(a.band, a.Hp - p0);
    const int nconv = 2 * npr + 1;                               // conv rows [2 * p0, 2 * p0 + nconv)
    const int S = a.stride, k = a.k, kk = k * k;
    const int rows_in = (nconv - 1) * S + k, cols_in = (a.Wo - 1) * S + k, plane = rows_in * cols_in;
    const int iy0 = 2 * p0 * S - 2;                              // input row of staged row 0 (padding 2)
    const int ppb = nconv * a.Wo, total = nb * ppb;
    float* s_w = smem;                                           // [cin_chunk][k * k][CO]
    float* s_in = smem + (size_t)a.cin_chunk * kk * CO;          // [nb][cc][rows_in][cols_in], then the conv tile

    float acc[ITEMS][4];
#pragma unroll
    for (int it = 0; it < ITEMS; ++it)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[it][c] = 0.0f;

    pdl_wait();                                                  // the input comes from the previous kernel
    for (int c0 = 0; c0 < a.cin; c0 += a.cin_chunk) {
        const int cc = min(a.cin_chunk, a.cin - c0);
        __syncthreads();
        for (int i = threadIdx.x; i < cc * kk * CO; i += blockDim.x) {
            const int co = i % CO, r = i / CO;                   // r = ci * k * k + tap
            s_w[i] = co < cov ? a.w[(size_t)(c0 * kk + r) * a.cout + co0 + co] : 0.0f;
        }
        for (int i = threadIdx.x; i < nb * cc * plane; i += blockDim.x) {
            const int x = i % cols_in, y = (i / cols_in) % rows_in, ci = (i / plane) % cc, b = i / (plane * cc);
            const int yi = iy0 + y, xi = x - 2;
            float v = 0.0f;
            if (yi >= 0 && yi < a.H && xi >= 0 && xi < a.W) v = a.in[(((size_t)(b0 + b) * a.cin + c0 + ci) * a.H + yi) * a.W + xi];
            s_in[i] = v;
        }
        __syncthreads();
        int base[ITEMS];
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) {
            const int pix = lane + it * lanes;
            base[it] = 0;                                        // an idle item computes on row 0 and is never stored
            if (pix < total) {
                const int b = pix / ppb, r = pix % ppb, y = r / a.Wo, x = r % a.Wo;
                base[it] = b * cc * plane + y * S * cols_in + x * S;
            }
        }
        for (int ci = 0; ci < cc; ++ci) {
            for (int ky = 0; ky < k; ++ky) {
                const float* wr = s_w + (ci * kk + ky * k) * CO + cg * 4;
                const float* xr = s_in + ci * plane + ky * cols_in;
                for (int kx = 0; kx < k; ++kx) {
                    const float4 w4 = *reinterpret_cast<const float4*>(wr + kx * CO);
#pragma unroll
                    for (int it = 0; it < ITEMS; ++it) {
                        const float xv = xr[base[it] + kx];
                        acc[it][0] = fmaf(xv, w4.x, acc[it][0]);
                        acc[it][1] = fmaf(xv, w4.y, acc[it][1]);
                        acc[it][2] = fmaf(xv, w4.z, acc[it][2]);
                        acc[it][3] = fmaf(xv, w4.w, acc[it][3]);
                    }
                }
            }
        }
    }
    // ---- conv tile (bias, ReLU) in shared memory, over the staged input
    __syncthreads();
    float* s_conv = s_in;                                        // [nb][CO][nconv][Wo]
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
        const int pix = lane + it * lanes;
        if (pix >= total) break;
        const int b = pix / ppb, r = pix % ppb, y = r / a.Wo, x = r % a.Wo;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int co = cg * 4 + c;
            const float bias = co < cov ? a.bias[co0 + co] : 0.0f;
            s_conv[((b * CO + co) * nconv + y) * a.Wo + x] = fmaxf(acc[it][c] + bias, 0.0f);
        }
    }
    __syncthreads();
    // ---- MaxPool2d(3, 2): to global memory, or to shared memory for the average
    float* s_pool = s_conv + nb * CO * nconv * a.Wo;            // [nb][CO][Hp][Wp] (average epilogue: npr = Hp)
    for (int i = threadIdx.x; i < nb * cov * npr * a.Wp; i += blockDim.x) {
        const int j = i % a.Wp, py = (i / a.Wp) % npr, co = (i / (a.Wp * npr)) % cov, b = i / (a.Wp * npr * cov);
        const float* src = s_conv + ((b * CO + co) * nconv + 2 * py) * a.Wo + 2 * j;
        float m = src[0];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) m = fmaxf(m, src[dy * a.Wo + dx]);
        if (a.avg_h) s_pool[((b * CO + co) * a.Hp + py) * a.Wp + j] = m;
        else a.out[(((size_t)(b0 + b) * a.cout + co0 + co) * a.Hp + p0 + py) * a.Wp + j] = m;
    }
    if (!a.avg_h) return;
    __syncthreads();
    // ---- AdaptiveAvgPool2d: bin [floor(i * In / Out), ceil((i + 1) * In / Out)) per dimension (upsamples when In < Out)
    const int ah = a.avg_h, aw = a.avg_w;
    for (int i = threadIdx.x; i < nb * cov * ah * aw; i += blockDim.x) {
        const int ox = i % aw, oy = (i / aw) % ah, co = (i / (aw * ah)) % cov, b = i / (aw * ah * cov);
        const int ys = oy * a.Hp / ah, ye = ((oy + 1) * a.Hp + ah - 1) / ah;
        const int xs = ox * a.Wp / aw, xe = ((ox + 1) * a.Wp + aw - 1) / aw;
        const float* src = s_pool + (b * CO + co) * a.Hp * a.Wp;
        float s = 0.0f;
        for (int y = ys; y < ye; ++y)
            for (int x = xs; x < xe; ++x) s = __fadd_rn(s, src[y * a.Wp + x]);
        a.out[(((size_t)(b0 + b) * a.cout + co0 + co) * ah + oy) * aw + ox] = __fdiv_rn(s, (float)((ye - ys) * (xe - xs)));
    }
}

constexpr size_t kStemSmemBudget = 112 * 1024;     // two CTAs per SM

int round4(int x) { return (x + 3) & ~3; }

// floats of shared memory of a stage tile
size_t stage_floats(const CnnStagePlan& p, int co, int band, int boards, int chunk, bool avg) {
    const int nconv = 2 * band + 1;
    const size_t plane = (size_t)((nconv - 1) * p.stride + p.k) * ((p.Wo - 1) * p.stride + p.k);
    const size_t staged = (size_t)boards * chunk * plane;
    const size_t tiles = (size_t)boards * co * nconv * p.Wo + (avg ? (size_t)boards * co * p.Hp * p.Wp : 0);
    return (size_t)chunk * p.k * p.k * co + std::max(staged, tiles);
}

bool plan_stage(int n, int cin, int cout, int H, int W, int k, int S, bool avg, int sm_count, const char* conv, const char* pool,
                CnnStagePlan* p, std::string* err) {
    *p = CnnStagePlan{};
    p->cin = cin; p->cout = cout; p->H = H; p->W = W; p->k = k; p->stride = S;
    if (H + 4 < k || W + 4 < k) {
        *err = std::string(conv) + ": kernel " + std::to_string(k) + " x " + std::to_string(k) + " is larger than the padded input (" +
               std::to_string(H) + " x " + std::to_string(W) + " + padding 2)";
        return false;
    }
    p->Ho = (H + 4 - k) / S + 1; p->Wo = (W + 4 - k) / S + 1;
    p->Hp = p->Ho >= 3 ? (p->Ho - 3) / 2 + 1 : 0;
    p->Wp = p->Wo >= 3 ? (p->Wo - 3) / 2 + 1 : 0;
    if (p->Hp < 1) { *err = std::string(pool) + " output is 0 rows (" + std::to_string(p->Ho) + " conv rows)"; return false; }
    if (p->Wp < 1) { *err = std::string(pool) + " output is 0 columns (" + std::to_string(p->Wo) + " conv columns)"; return false; }
    const size_t budget = kStemSmemBudget / 4;
    const int tiles0 = (cout + 63) / 64;
    for (int co = std::min(64, round4((cout + tiles0 - 1) / tiles0));; co = std::max(4, round4(co / 2))) {
        const int cgs = co / 4, lanes = kCnnStemThreads / cgs;
        const int co_tiles = (cout + co - 1) / co;
        // the band: as many pooled rows as four items per thread cover (all of them with the average epilogue)
        int band = p->Hp;
        if (!avg) while (band > 1 && (2 * band + 1) * p->Wo > lanes * 4) --band;
        if ((2 * band + 1) * p->Wo <= lanes * 16) {
            int nb = std::max(1, std::min(std::min(n, 32), lanes * 4 / ((2 * band + 1) * p->Wo)));
            // spread the batch: two CTAs per SM where it is large enough, then bands for small batches
            while (nb > 1 && (long)((n + nb - 1) / nb) * co_tiles * ((p->Hp + band - 1) / band) < 2L * sm_count) nb = (nb + 1) / 2;
            if (!avg)
                while (band > 1 && (long)((n + nb - 1) / nb) * co_tiles * ((p->Hp + band - 1) / band) < sm_count) band = (band + 1) / 2;
            for (;;) {
                int chunk = cin;
                while (chunk > 1 && stage_floats(*p, co, band, nb, chunk, avg) > budget) chunk = (chunk + 1) / 2;
                if (stage_floats(*p, co, band, nb, chunk, avg) <= budget) {
                    const int need = (nb * (2 * band + 1) * p->Wo + lanes - 1) / lanes;
                    int items = 1;
                    while (items < need) items *= 2;
                    p->co_tile = co; p->band = band; p->bands = (p->Hp + band - 1) / band; p->boards = nb; p->cin_chunk = chunk;
                    p->items = items; p->threads = cgs * lanes;
                    p->grid = dim3((n + nb - 1) / nb, co_tiles, p->bands);
                    p->smem = stage_floats(*p, co, band, nb, chunk, avg) * 4;
                    return true;
                }
                if (nb > 1) nb = (nb + 1) / 2;
                else if (!avg && band > 1) band = (band + 1) / 2;
                else break;
            }
        }
        if (co == 4) break;
    }
    *err = std::string(conv) + " + " + pool + ": the tile of one board does not fit in shared memory (" + std::to_string(p->Ho) +
           " x " + std::to_string(p->Wo) + " conv output, kernel " + std::to_string(k) + ")";
    return false;
}

template <int ITEMS>
cudaError_t launch_stage(const CnnStageArgs& a, const CnnStagePlan& p, cudaStream_t stream) {
    static size_t attr = 0;
    if (attr < p.smem) {
        cudaError_t e = cudaFuncSetAttribute(cnn_stage_kernel<ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
        if (e != cudaSuccess) return e;
        attr = p.smem;
    }
    cudaError_t e = launch_chained(cnn_stage_kernel<ITEMS>, p.grid, dim3(p.threads), p.smem, stream, a);
    return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t run_stage(const CnnStagePlan& p, const float* in, float* out, const float* w, const float* bias, int n, int ah, int aw,
                      cudaStream_t stream) {
    CnnStageArgs a{};
    static_cast<CnnStagePlan&>(a) = p;
    a.in = in; a.out = out; a.w = w; a.bias = bias; a.n = n; a.avg_h = ah; a.avg_w = aw;
    switch (p.items) {
        case 1: return launch_stage<1>(a, p, stream);
        case 2: return launch_stage<2>(a, p, stream);
        case 4: return launch_stage<4>(a, p, stream);
        case 8: return launch_stage<8>(a, p, stream);
        case 16: return launch_stage<16>(a, p, stream);
    }
    return cudaErrorInvalidValue;
}

}  // namespace

bool cnn_stem_plan(int n, int in, int C, int H, int W, int sm_count, CnnStemPlan* p, std::string* err) {
    *p = CnnStemPlan{};
    if (n < 1 || in < 1 || C < 1 || H < 1 || W < 1 || sm_count < 1) { *err = "cnn stem: empty shape"; return false; }
    p->h = (H + 15) / 16; p->w = (W + 15) / 16;
    p->mid = (in + C) / 2;
    if (!plan_stage(n, in, p->mid, H, W, 2 * p->h, 4, false, sm_count, "conv1", "pool1", &p->s[0], err)) return false;
    return plan_stage(n, p->mid, C, p->s[0].Hp, p->s[0].Wp, 5, 1, true, sm_count, "conv2", "pool2", &p->s[1], err);
}

void cnn_stem_plan_export(const CnnStemPlan& p, int64_t* out) {
    for (int i = 0; i < kCnnPlanLen; ++i) out[i] = 0;
    out[0] = p.h; out[1] = p.w; out[2] = p.mid;
    for (int s = 0; s < 2; ++s) {
        const CnnStagePlan& q = p.s[s];
        const int64_t v[16] = {q.k, q.stride, q.Ho, q.Wo, q.Hp, q.Wp, q.co_tile, q.band, q.bands, q.boards, q.cin_chunk, q.items,
                               q.threads, q.grid.x, q.grid.y, (int64_t)q.smem};
        for (int i = 0; i < 16; ++i) out[3 + 16 * s + i] = v[i];
    }
}

CnnStemWeights cnn_stem_pack(const float* w1, const float* b1, const float* w2, const float* b2, int in, int mid, int C, int k,
                             std::vector<float>& blob) {
    // [cout][cin][kk] -> [cin][kk][cout] (a bias is the case cin = kk = 1)
    auto put = [&](const float* w, int cout, int cin, int kk) {
        const size_t off = blob.size();
        blob.resize(off + (size_t)cin * kk * cout);
        for (int co = 0; co < cout; ++co)
            for (int ci = 0; ci < cin; ++ci)
                for (int t = 0; t < kk; ++t) blob[off + ((size_t)ci * kk + t) * cout + co] = w[((size_t)co * cin + ci) * kk + t];
        while (blob.size() % 4) blob.push_back(0.0f);
        return off;
    };
    CnnStemWeights o;
    o.w1 = put(w1, mid, in, k * k); o.b1 = put(b1, mid, 1, 1);
    o.w2 = put(w2, C, mid, 25); o.b2 = put(b2, C, 1, 1);
    return o;
}

cudaError_t cnn_stem_launch(const CnnStemPlan& p, const float* blob, const CnnStemWeights& w, const float* x, float* pooled,
                            float* out, int n, cudaStream_t stream) {
    cudaError_t e = run_stage(p.s[0], x, pooled, blob + w.w1, blob + w.b1, n, 0, 0, stream);
    if (e != cudaSuccess) return e;
    return run_stage(p.s[1], pooled, out, blob + w.w2, blob + w.b2, n, p.h, p.w, stream);
}

int cnn_stem_debug(int n, int in, int C, int H, int W, const float* x, const float* w1, const float* b1, const float* w2,
                   const float* b2, float* out, int64_t* plan, int sm_count, std::string* err) {
    CnnStemPlan p;
    if (!cnn_stem_plan(n, in, C, H, W, sm_count, &p, err)) return MZ_EUNSUPPORTED;
    std::vector<float> blob;
    const CnnStemWeights w = cnn_stem_pack(w1, b1, w2, b2, in, p.mid, C, 2 * p.h, blob);
    const size_t nx = (size_t)n * in * H * W, np = (size_t)n * p.mid * p.s[0].Hp * p.s[0].Wp, no = (size_t)n * C * p.h * p.w;
    float *d_blob = nullptr, *d_x = nullptr, *d_p = nullptr, *d_o = nullptr;
    auto cleanup = [&]() { for (float* q : {d_blob, d_x, d_p, d_o}) if (q) cudaFree(q); };
    if (cudaMalloc(&d_blob, blob.size() * 4) != cudaSuccess || cudaMalloc(&d_x, nx * 4) != cudaSuccess ||
        cudaMalloc(&d_p, np * 4) != cudaSuccess || cudaMalloc(&d_o, no * 4) != cudaSuccess) {
        cleanup(); *err = "allocation failed"; return MZ_ENOMEM;
    }
    cudaMemcpy(d_blob, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_x, x, nx * 4, cudaMemcpyHostToDevice);
    cudaMemset(d_p, 0xFF, np * 4);                     // NaN: an element the kernels do not write cannot pass a test
    cudaMemset(d_o, 0xFF, no * 4);
    cudaError_t e = cnn_stem_launch(p, d_blob, w, d_x, d_p, d_o, n, nullptr);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, d_o, no * 4, cudaMemcpyDeviceToHost);
    cleanup();
    if (plan) cnn_stem_plan_export(p, plan);
    if (e != cudaSuccess) { *err = std::string("cnn stem: ") + cudaGetErrorString(e); return MZ_ECUDA; }
    return MZ_OK;
}

}  // namespace mz
