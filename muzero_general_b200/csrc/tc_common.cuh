// Device helpers shared by the tensor-core tower kernels (conv_tc.cu, conv_x3.cu, conv_wide.cu, conv_wide256.cu):
// mbarriers, bulk copies (TMA unit), warpgroup MMAs (wgmma) with shared-memory matrix descriptors, fp16 packing and
// splitting, distributed shared memory of a cluster.
#pragma once
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "common.cuh"

namespace mz {
namespace tc {

MZ_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

MZ_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
MZ_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
MZ_DEVINL void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
MZ_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    } while (!done);
}
MZ_DEVINL void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// wgmma matrix descriptor words shared by every A / B operand (K-major SWIZZLE_128B, SBO = 1024 B between 8-row groups):
// lo = start address / 16 | LBO field 1 (unused for K-major swizzled operands), hi = SBO / 16 | layout type 1 (128B
// swizzle, bits 62-63).  The 128B swizzle is applied on absolute shared-memory address bits, so row-shifted tap windows
// need no base_offset (tests/test_conv_gpu.py is exact only if that holds).
constexpr uint32_t kDescLoFlags = 1u << 16;
constexpr uint32_t kDescHi = ((1024u >> 4) & 0x3FFFu) | (1u << 30);

// shared -> global bulk copy (TMA unit), tracked by the thread's bulk async-group
MZ_DEVINL void bulk_s2g(void* gdst, uint32_t ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}

MZ_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
MZ_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
MZ_DEVINL void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T on one warpgroup: fp16 operands from shared memory (descriptor low words,
// K-major), fp32 accumulators in registers.  Thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and
// columns 8 j + 2 (t % 4) (+ 1): d[4 j + 2 h + e] = D[row + 8 h][8 j + 2 (t % 4) + e].
MZ_DEVINL void wgmma_m64n64k16(float* d, uint32_t a_lo, uint32_t b_lo, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        ".reg .b64 da, db;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "mov.b64 da, {%32, %35};\n\t"
        "mov.b64 db, {%33, %35};\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, da, db, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a_lo), "r"(b_lo), "r"(accumulate), "r"(kDescHi)
        : "memory");
}

// barrier over the 128 threads of warpgroup wg (named barrier 1 + wg; 0 is __syncthreads)
MZ_DEVINL void warpgroup_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

MZ_DEVINL void wgmma_wait_one() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// fp32 -> (x_h, x_l = (v - x_h) 2^11) as the x3 towers on dense boards split their inputs (conv_wide.cu,
// conv_wide256.cu): both halves saturate to the finite fp16 range
MZ_DEVINL void split_store(unsigned char* hi, unsigned char* lo, float v) {
    const float s = fminf(fmaxf(v, -65504.0f), 65504.0f);
    const __half h = __float2half_rn(s);
    *reinterpret_cast<__half*>(hi) = h;
    *reinterpret_cast<__half*>(lo) = __float2half_rn(fminf(fmaxf((v - __half2float(h)) * 2048.0f, -65504.0f), 65504.0f));
}

// distributed shared memory of a cluster (the CTA pairs of conv_wide.cu and conv_wide256.cu)
MZ_DEVINL uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
MZ_DEVINL uint32_t map_to_cta(uint32_t addr, uint32_t rank) {     // my shared::cta address -> the same offset in CTA `rank`
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
MZ_DEVINL void st_cluster_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
MZ_DEVINL void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// two fp32 -> packed fp16x2, round to nearest even, saturating to the finite range
MZ_DEVINL uint32_t pack_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
MZ_DEVINL float2 unpack_f16x2(uint32_t v) {
    __half2 h = *reinterpret_cast<__half2*>(&v);
    return __half22float2(h);
}


}  // namespace tc
}  // namespace mz
