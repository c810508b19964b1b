// Attention dropout inside the fused wgmma attention kernels: the kernel bodies of attention_sm90.cuh instantiated with
// kDrop = true, which apply the dropout mask where the probabilities live in registers, so that no score or probability
// buffer reaches HBM.  Same tiles, pipelines and work items as attention_sm90.cu (see its header).  These kernels are
// instantiated in their own translation unit: compiled next to them, the plain kernels' SASS would not stay as it is.
//
// Mask: that of the stand-alone dropout kernel (dropout.cuh) applied to the probabilities laid out as [B*H, N, ldp]
// with ldp = pad8(N): element (bh, query q, key k) is chunk k % 8 of Philox vector (bh * N + q) * ldp / 8 + k / 8.  A run
// with attention dropout therefore keeps and drops the same elements on the fused and on the un-fused path.
//   forward : the row sums and the log-sum-exp are those of the undropped P; P o M * s feeds O += P V.
//   backward: P is rebuilt from the log-sum-exp; dV += (P o M s)^T dO and dS = P o (dP o M s - delta), where delta =
//             rowsum(dO o O) is unchanged because O is the dropped output.
// Each of the 512 (row, 8-key) Philox vectors of a 64 x 64 tile is evaluated once per CTA (4 per thread) while the tile's
// MMAs run, and its keep bits reach the lanes that hold its elements through shuffles.
//
// These kernels are call-free (silent barrier waits, no printf), so ptxas keeps their wgmma batches pipelined.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <stdexcept>

#include "attention_sm90.cuh"
#include "attention_sm90.h"

namespace b200 {

namespace {

template <int HD>
__global__ void __launch_bounds__(kAttnThreads) attn_fwd_drop_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                                                         const __grid_constant__ CUtensorMap tmap_k,
                                                                         const __grid_constant__ CUtensorMap tmap_v,
                                                                         const AttnParams p, const DropParams d) {
    attn_fwd_body<HD, true>(tmap_q, tmap_k, tmap_v, p, d);
}

template <int HD, int kRole>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_drop_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                                                         const __grid_constant__ CUtensorMap tmap_k,
                                                                         const __grid_constant__ CUtensorMap tmap_v,
                                                                         const __grid_constant__ CUtensorMap tmap_do,
                                                                         const BwdParams p, const DropParams d) {
    attn_bwd_body<HD, kRole, true>(tmap_q, tmap_k, tmap_v, tmap_do, p, d);
}

}  // namespace

void attention_fwd_drop(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, int B, int N, int H,
                        int hd, float drop_p, uint64_t drop_key, cudaStream_t stream) {
    if (!shape_ok(N, hd)) throw std::runtime_error("attention_fwd: unsupported (N, head_dim)");
    const DropParams d = make_drop(drop_p, drop_key, "attention_fwd");
    run_fwd<true>(qkv, ld_qkv, out, lse, nullptr, 0, B, N, H, hd, d, stream);
}

void attention_bwd_drop(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do,
                        const float* lse, const float* delta, __nv_bfloat16* dqkv, int B, int N, int H, int hd,
                        float* colsum, float drop_p, uint64_t drop_key, cudaStream_t stream) {
    if (!shape_ok(N, hd)) throw std::runtime_error("attention_bwd: unsupported (N, head_dim)");
    const DropParams d = make_drop(drop_p, drop_key, "attention_bwd");
    run_bwd<true>(qkv, ld_qkv, dout, ld_do, lse, delta, dqkv, B, N, H, hd, colsum, d, stream);
}

}  // namespace b200
