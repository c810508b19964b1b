// Philox-4x32-10 dropout mask shared by the stand-alone dropout kernel (elementwise.cu) and the fused attention kernels
// (attention_sm90.cu), so that both keep or drop exactly the same elements for the same key.
//
// Element e of a dropped tensor belongs to the 16-byte vector i = e / 8; philox4x32_10(lo32(i), hi32(i), key) gives
// 8 x 16 random bits, chunk c = e % 8 is (r[c >> 1] >> 16 * (c & 1)) & 0xFFFF, and the element is kept iff that chunk is
// >= dropout_thresh16(p).  Kept values are scaled by dropout_scale(thresh).
#pragma once
#include <cstdint>

namespace b200 {

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1, uint32_t (&out)[4]) {
    uint32_t c2 = 0x5eed5eedu, c3 = 0x0b200b20u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c0, out[1] = c1, out[2] = c2, out[3] = c3;
}

// Drop probability p in [0, 1) -> 16-bit keep threshold, and the scale of the kept values.
inline uint32_t dropout_thresh16(float p) { return static_cast<uint32_t>(p * 65536.0f + 0.5f); }
inline float dropout_scale(uint32_t thresh16) { return 1.0f / (1.0f - static_cast<float>(thresh16) / 65536.0f); }

// Keep bits of the 8 elements of vector i: bit c set iff element 8 * i + c is kept.
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t i, uint32_t key_lo, uint32_t key_hi, uint32_t thresh16) {
    uint32_t r[4];
    philox4x32_10(static_cast<uint32_t>(i), static_cast<uint32_t>(i >> 32), key_lo, key_hi, r);
    uint32_t bits = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) bits |= static_cast<uint32_t>(((r[c >> 1] >> ((c & 1) * 16)) & 0xFFFFu) >= thresh16) << c;
    return bits;
}

}  // namespace b200
