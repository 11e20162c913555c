// Philox4x32-10 (Salmon et al. SC'11) and the keyed draws of the device loop; mirrored in oracle/philox.py.
// This header is also compiled by NVRTC as part of the prelude of user environments (user_env.cuh), so it includes
// nothing: the includer provides uint32_t, uint64_t, int64_t and MZ_DEVINL.
#pragma once

namespace mz {

constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u;
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u;
constexpr uint32_t kTagTie = 0x7169E001u, kTagNoise = 0x7169E002u, kTagAction = 0x7169E003u;
constexpr uint32_t kTagReset = 0x7169E004u;      // CartPole's reset state
constexpr uint32_t kTagOpponent = 0x7169E005u;   // the random default of test-mode opponents
constexpr uint32_t kTagCard = 0x7169E006u;       // Twenty-One's cards
constexpr uint32_t kTagPlace = 0x7169E007u;      // Gridworld's placement

struct Philox4 { uint32_t x, y, z, w; };

MZ_DEVINL Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t p0h = __umulhi(kPhiloxM0, c0), p0l = kPhiloxM0 * c0;
        const uint32_t p1h = __umulhi(kPhiloxM1, c2), p1l = kPhiloxM1 * c2;
        c0 = p1h ^ c1 ^ k0; c1 = p1l;
        c2 = p0h ^ c3 ^ k1; c3 = p0l;
        k0 += kPhiloxW0; k1 += kPhiloxW1;
    }
    return Philox4{c0, c1, c2, c3};
}

// A uniform in [0, 1) with 53 random bits, keyed (seed, game, move, c2, tag): counter (game, move, c2, game >> 32),
// key (seed, (seed >> 32) ^ tag)
MZ_DEVINL double philox_uniform53(uint64_t seed, int64_t game, int move, uint32_t c2, uint32_t tag) {
    const Philox4 r = philox4x32_10((uint32_t)game, (uint32_t)move, c2, (uint32_t)((uint64_t)game >> 32),
                                    (uint32_t)seed, (uint32_t)(seed >> 32) ^ tag);
    // 53 random bits like numpy's random_sample: (a >> 5) * 2^26 + (b >> 6)
    return ((double)(r.x >> 5) * 67108864.0 + (double)(r.y >> 6)) * (1.0 / 9007199254740992.0);
}

}  // namespace mz
