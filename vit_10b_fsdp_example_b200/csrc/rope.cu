// Rotary position embedding (2-D axial RoPE, EVA-02 / timm RotaryEmbeddingCat) on the packed [rows, 3D] qkv buffer.
// See rope.h for the layout and the tables.
//
// One memory-bound pass.  A thread owns one 16-byte vector (4 interleaved pairs, inside one head since hd % 8 == 0) of
// a column strip and walks a slab of rows, kRopeRows rows in flight; consecutive threads read consecutive vectors of a
// row.  The rotation runs in fp32 on the bf16 inputs and rounds once.  The backward also sums its columns in registers
// and adds them with one atomic per column per CTA.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <climits>
#include <cstdint>
#include <stdexcept>
#include <string>

#include "ptx.cuh"
#include "rope.cuh"

namespace b200 {

namespace {

constexpr int kRopeThreads = 256;
constexpr int kRopeRows = 4;      // rows whose loads are in flight together
constexpr int kRopeMaxHd = 256;   // the range qk_norm takes

__device__ __forceinline__ void rope_unpack8(const uint4& v, float (&f)[8]) {
    f[0] = bf16_lo(v.x), f[1] = bf16_hi(v.x), f[2] = bf16_lo(v.y), f[3] = bf16_hi(v.y);
    f[4] = bf16_lo(v.z), f[5] = bf16_hi(v.z), f[6] = bf16_lo(v.w), f[7] = bf16_hi(v.w);
}
__device__ __forceinline__ uint4 rope_pack8(const float (&f)[8]) {
    uint4 v;
    v.x = pack_bf16x2(f[0], f[1]), v.y = pack_bf16x2(f[2], f[3]);
    v.z = pack_bf16x2(f[4], f[5]), v.w = pack_bf16x2(f[6], f[7]);
    return v;
}

// Forward (kBwd false): y[:, 0:8 nvec) = x with the q / k vectors (idx < nvec_rot) of patch rows rotated by R.  In place
// (y == x) nvec == nvec_rot and only rotated vectors are stored; out of place everything in [0, 8 nvec) is stored.
// Backward (kBwd true, y == x, nvec == nvec_rot): R^T in place, and colsum += column sums of the stored values.
// x / y are not __restrict__: in place, every element is read by the thread that later overwrites it, and by no other.
template <bool kBwd>
__global__ void __launch_bounds__(kRopeThreads) rope_kernel(const __nv_bfloat16* x, int64_t ld, __nv_bfloat16* y,
                                                            int64_t ld_y, RopeArgs r, int rows, int hd, int nvec_rot,
                                                            int nvec, int rows_per_cta, float* __restrict__ colsum) {
    const int idx = blockIdx.x * kRopeThreads + threadIdx.x;
    if (idx >= nvec) return;
    const bool rot = idx < nvec_rot;
    const bool in_place = x == y;
    const int half = hd / 2;
    const int p = (idx * 8) % hd / 2;  // first pair of this vector in its head
    const int r0 = blockIdx.y * rows_per_cta;
    const int r1 = min(rows, r0 + rows_per_cta);
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    for (int t = r0; t < r1; t += kRopeRows) {
        uint4 v[kRopeRows];
        int n[kRopeRows];
#pragma unroll
        for (int u = 0; u < kRopeRows; ++u) {
            const bool ok = t + u < r1;
            v[u] = ok ? reinterpret_cast<const uint4*>(x + static_cast<int64_t>(t + u) * ld)[idx] : make_uint4(0, 0, 0, 0);
            n[u] = ok && rot ? rope_row(r, t + u) : -1;
        }
#pragma unroll
        for (int u = 0; u < kRopeRows; ++u) {
            if (t + u >= r1) break;
            uint4 o = v[u];
            if (n[u] >= 0) {
                float f[8];
                rope_unpack8(o, f);
                rope_rotate<kBwd>(f, r, n[u], half, p);
                o = rope_pack8(f);
            }
            if (n[u] >= 0 || !in_place)
                reinterpret_cast<uint4*>(y + static_cast<int64_t>(t + u) * ld_y)[idx] = o;
            if (kBwd) {
                float f[8];
                rope_unpack8(o, f);  // the sums are those of the rounded gradient the GEMMs consume
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[q] += f[q];
            }
        }
    }
    if (kBwd) {
#pragma unroll
        for (int q = 0; q < 8; ++q) atomicAdd(colsum + idx * 8 + q, acc[q]);
    }
}

inline void check_launch_rope(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

int sm_count_rope() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    }
    return n;
}

void fail(const char* what, const std::string& msg) { throw std::runtime_error(std::string(what) + ": " + msg); }

void check_rope_matrix(const char* what, const char* name, const void* p, int64_t ld, int64_t width) {
    if ((reinterpret_cast<uintptr_t>(p) & 15) || ld % 8 != 0)
        fail(what, std::string(name) + " must be 16-byte aligned with a leading dimension that is a multiple of 8 "
                   "elements (16 bytes), got ld " + std::to_string(ld));
    if (ld < width)
        fail(what, std::string(name) + " leading dimension " + std::to_string(ld) + " is narrower than 3 * H * hd = " +
                   std::to_string(width));
}

}  // namespace

void check_rope_args(const char* what, const RopeArgs& r, int B, int H, int hd) {
    if (hd % 8 != 0 || hd < 8 || hd > kRopeMaxHd)
        fail(what, "head dim must be a multiple of 8 in [8, 256] (hd % 8 == 0 and 8 <= hd <= 256), got " +
                   std::to_string(hd));
    if (B < 1 || H < 1) fail(what, "need B >= 1 and H >= 1");
    if (r.tokens < 1 || r.prefix < 0 || r.prefix > r.tokens)
        fail(what, "need tokens per image T >= 1 and 0 <= P <= T, got T " + std::to_string(r.tokens) + ", P " +
                   std::to_string(r.prefix));
    if (static_cast<int64_t>(B) * r.tokens > INT_MAX)
        fail(what, "rows B * T = " + std::to_string(static_cast<int64_t>(B) * r.tokens) + " overflow 32 bits");
    if (static_cast<int64_t>(r.n_tab) * (hd / 2) > INT_MAX)
        fail(what, "table rows * hd / 2 overflow 32 bits");
    if (!r.cos || !r.sin || ((reinterpret_cast<uintptr_t>(r.cos) | reinterpret_cast<uintptr_t>(r.sin)) & 15))
        fail(what, "cos / sin tables must be 16-byte aligned fp32 [N, hd / 2]");
    const int K = r.tokens - r.prefix;
    if (K > r.n_tab)
        fail(what, "table has " + std::to_string(r.n_tab) + " rows but every image has T - P = " + std::to_string(K) +
                   " patch tokens (the table must cover the full grid)");
}

void rope_fwd(const __nv_bfloat16* qkv, int64_t ld, __nv_bfloat16* out, int64_t ld_out, const RopeArgs& rope, int B,
              int H, int hd, cudaStream_t stream) {
    check_rope_args("rope_fwd", rope, B, H, hd);
    const int64_t width = 3 * static_cast<int64_t>(H) * hd;
    check_rope_matrix("rope_fwd", "qkv", qkv, ld, width);
    check_rope_matrix("rope_fwd", "out", out, ld_out, width);
    const bool in_place = out == qkv;
    if (in_place && ld_out != ld) fail("rope_fwd", "in place needs ld_out == ld");
    const int rows = B * rope.tokens;
    const int nvec_rot = static_cast<int>(2 * width / 3 / 8);
    const int nvec = in_place ? nvec_rot : static_cast<int>(width / 8);
    const int gx = (nvec + kRopeThreads - 1) / kRopeThreads;
    const int slabs = std::max(1, std::min(std::min(rows, 65535), sm_count_rope() * 8 / gx));
    const int rows_per = (rows + slabs - 1) / slabs;
    const dim3 grid(gx, (rows + rows_per - 1) / rows_per);
    rope_kernel<false><<<grid, kRopeThreads, 0, stream>>>(qkv, ld, out, ld_out, rope, rows, hd, nvec_rot, nvec,
                                                          rows_per, nullptr);
    check_launch_rope("rope_fwd");
}

void rope_bwd(__nv_bfloat16* dqkv, int64_t ld, const RopeArgs& rope, int B, int H, int hd, float* colsum,
              cudaStream_t stream) {
    check_rope_args("rope_bwd", rope, B, H, hd);
    const int64_t width = 3 * static_cast<int64_t>(H) * hd;
    check_rope_matrix("rope_bwd", "dqkv", dqkv, ld, width);
    const int rows = B * rope.tokens;
    const int nvec = static_cast<int>(2 * width / 3 / 8);
    const int gx = (nvec + kRopeThreads - 1) / kRopeThreads;
    const int slabs = std::max(1, std::min(std::min(rows, 65535), sm_count_rope() * 8 / gx));
    const int rows_per = (rows + slabs - 1) / slabs;
    const dim3 grid(gx, (rows + rows_per - 1) / rows_per);
    rope_kernel<true><<<grid, kRopeThreads, 0, stream>>>(dqkv, ld, dqkv, ld, rope, rows, hd, nvec, nvec, rows_per,
                                                         colsum);
    check_launch_rope("rope_bwd");
}

}  // namespace b200
