// NVLink / NVSwitch collectives over symmetric (peer-mapped) memory, written directly against raw
// peer / multicast pointers -- no NCCL on these paths.
//
// Every kernel here is a *light* CTA: 128 threads, <= 96 registers, no shared memory, many 16-byte requests in
// flight per thread, so that several fit one SM and a collective needs few SMs.  A resident GEMM CTA (gemm_sm90.cu)
// takes 224 KB of shared memory and 384 x 168 of the SM's 65536 registers, so a collective CTA never shares an SM
// with it: it is placed on an SM as a GEMM CTA retires.  How much of a collective hides under the GEMMs on H100 has
// not been measured.
//
//   p2p_all_gather      : sync-free pull of the peers' parameter shards straight into their final
//                         position in the gathered flat buffer (no copy-out pass).  Shards only change in
//                         the optimizer step, so no per-block flags are needed.
//   reduce_scatter      : ONE kernel per unit: publish "my gradients are complete" to every peer, wait for
//                         theirs, reduce this rank's slab (multimem.ld_reduce inside the NVSwitch, or peer
//                         pulls), apply 1/W, write the fp32 shard gradient (or run AdamW right there) and the
//                         sum-of-squares partial for the global grad norm, then publish "done reading" and wait
//                         until every peer is done too (the buffer may be overwritten afterwards).  No separate
//                         barrier launches; the flag waits are done by a single warp of the last CTA.
//   all_reduce          : same protocol, in-place mean over a replicated bf16 buffer (DDP mode): in-switch
//                         multimem.ld_reduce + multimem.st, or pull-reduce-push over peer pointers.
//   signal_barrier      : device-side barrier through flags in symmetric memory (st.release.sys /
//                         ld.acquire.sys), monotonically increasing sequence numbers, bounded spin.
//   allreduce_scalars   : W x K floats exchanged through symmetric scratch (grad-norm^2, loss, max time).
//
// Capability parity: XLA all_gather / reduce_scatter / all_reduce emitted by XlaFullyShardedDataParallel
// (reference run_vit_training.py:177-181, 261-270), xm.reduce_gradients (:273) and xm.mesh_reduce (:205).
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "comm.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kMaxWorld = 16;
constexpr int kCommThreads = 128;
constexpr int kAgUnroll = 8;   // 16 B loads in flight per thread (all-gather)
constexpr int kRsUnroll = 4;   // 16 B multimem / peer vectors in flight per thread (reduce-scatter, all-reduce)

struct PeerPtrs {
    uint64_t p[kMaxWorld];
};

__device__ __forceinline__ uint4 ld_stream_v4(const void* ptr) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(ptr)
                 : "memory");
    return r;
}
__device__ __forceinline__ void st_stream_v4(void* ptr, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(ptr), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}
// Streaming stores whose lines are the first to leave L2: the gathered parameters / reduced gradients are consumed
// milliseconds later, while the co-running GEMM lives off the A/B panels it keeps L2-resident.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void st_stream_v4_hint(void* ptr, const uint4& v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(ptr), "r"(v.x),
                 "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ uint4 ld_stream_v4_hint(const void* ptr, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(ptr), "l"(pol)
                 : "memory");
    return r;
}
__device__ __forceinline__ void st_release_sys(uint32_t* ptr, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(ptr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* ptr) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(ptr) : "memory");
    return v;
}
__device__ __forceinline__ float ld_relaxed_sys_f32(const float* ptr) {
    float v;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(ptr) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_f32(float* ptr, float v) {
    asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(ptr), "f"(v) : "memory");
}
// In-switch reduction of 8 bf16 values (fp32 accumulate) over all GPUs bound to the multicast object.
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc_ptr) {
    uint4 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(mc_ptr)
                 : "memory");
    return r;
}
// One store, delivered by the NVSwitch to the same offset on every GPU of the multicast object.
__device__ __forceinline__ void multimem_st_v4(void* mc_ptr, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_ptr), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

constexpr int64_t kAgChunkBytes = static_cast<int64_t>(kCommThreads) * kAgUnroll * 16;  // 16 KiB: one CTA pass
constexpr int64_t kRsChunkVecs = static_cast<int64_t>(kCommThreads) * kRsUnroll;        // 16 B vectors per chunk
constexpr int64_t kRsChunkElems = kRsChunkVecs * 8;                                     // in bf16 elements

// ------------------------------------------------------------------------------------------------------------
// Cross-GPU flag protocol shared by reduce_scatter / all_reduce.
//   flags   : every rank's symmetric flag region, uint32 [slot][kMaxWorld]
//   seq_dev : device-resident call counters (every rank issues the same sequence of collectives, so the
//             counters agree without communication; keeping them on the device makes launches graph-replayable)
//   cta_ctr : zero-initialised device word, last-CTA detection
// ------------------------------------------------------------------------------------------------------------
struct SyncArgs {
    PeerPtrs flags;
    int rank, world;
    int slot_ready, slot_done;
    uint32_t* seq_dev;
    int counter_idx;
    uint32_t* cta_ctr;
};

__device__ __forceinline__ void spin_until(const uint32_t* flag, uint32_t seq, int rank, int peer, const char* what) {
    uint32_t spins = 0;
    // Sequence numbers only grow; signed distance handles wrap-around.
    while (static_cast<int32_t>(ld_acquire_sys(flag) - seq) < 0) {
        __nanosleep(64);
        if (++spins > (1u << 26)) {
            printf("[b200] %s timeout: rank %d waiting for peer %d seq %u\n", what, rank, peer, seq);
            __trap();
        }
    }
}

// Start of a collective: CTA 0 tells every peer that this rank's input buffer is complete (the kernel is
// stream-ordered after its producer), then every CTA waits until all peers have said the same.
__device__ __forceinline__ uint32_t sync_begin(const SyncArgs& s) {
    if (s.world <= 1) return 0;
    const uint32_t seq = s.seq_dev[s.counter_idx] + 1;
    const int t = threadIdx.x;
    if (t < s.world) {
        if (blockIdx.x == 0) {
            __threadfence_system();
            st_release_sys(reinterpret_cast<uint32_t*>(s.flags.p[t]) + s.slot_ready * kMaxWorld + s.rank, seq);
        }
        spin_until(reinterpret_cast<const uint32_t*>(s.flags.p[s.rank]) + s.slot_ready * kMaxWorld + t, seq, s.rank, t,
                   "collective (inputs ready)");
    }
    __syncthreads();
    return seq;
}

// End of a collective: the last CTA to finish tells every peer that this rank no longer touches their buffers and
// waits for the same from all of them; only one warp of one CTA stays resident for that wait.
__device__ __forceinline__ void sync_end(const SyncArgs& s, uint32_t seq) {
    if (s.world <= 1) return;
    __threadfence_system();  // this thread's stores (possibly to peers) are ordered before the "done" flag below
    __syncthreads();
    int last = 0;
    if (threadIdx.x == 0) {
        last = atomicAdd(s.cta_ctr, 1u) == gridDim.x - 1;
        __threadfence();
    }
    if (!__syncthreads_or(last)) return;
    const int t = threadIdx.x;
    if (t < s.world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<uint32_t*>(s.flags.p[t]) + s.slot_done * kMaxWorld + s.rank, seq);
        spin_until(reinterpret_cast<const uint32_t*>(s.flags.p[s.rank]) + s.slot_done * kMaxWorld + t, seq, s.rank, t,
                   "collective (peers done)");
    }
    __syncthreads();
    if (t == 0) {
        *s.cta_ctr = 0;
        s.seq_dev[s.counter_idx] = seq;
    }
}

// seg_table row (all-gather): [src_rank, src_off_bytes, dst_off_bytes, nbytes, chunk_prefix]
__global__ void __launch_bounds__(kCommThreads, 8) p2p_all_gather_kernel(PeerPtrs peers, uint8_t* __restrict__ out,
                                                                         const int64_t* __restrict__ seg, int nseg,
                                                                         int64_t total_chunks, int l2_hint) {
    int s = 0;
    const uint64_t pol = l2_evict_first_policy();
    for (int64_t c = blockIdx.x; c < total_chunks; c += gridDim.x) {
        while (s + 1 < nseg && seg[(s + 1) * 5 + 4] <= c) ++s;
        const int64_t* row = seg + s * 5;
        const int64_t off = (c - row[4]) * kAgChunkBytes;
        const int64_t nvec = min(kAgChunkBytes, row[3] - off) / 16;
        const uint8_t* src = reinterpret_cast<const uint8_t*>(peers.p[row[0]]) + row[1] + off;
        uint8_t* dst = out + row[2] + off;
        uint4 v[kAgUnroll];
#pragma unroll
        for (int u = 0; u < kAgUnroll; ++u) {
            const int64_t i = threadIdx.x + u * kCommThreads;
            if (i < nvec) v[u] = l2_hint ? ld_stream_v4_hint(src + i * 16, pol) : ld_stream_v4(src + i * 16);
        }
#pragma unroll
        for (int u = 0; u < kAgUnroll; ++u) {
            const int64_t i = threadIdx.x + u * kCommThreads;
            if (i < nvec) {
                if (l2_hint) st_stream_v4_hint(dst + i * 16, v[u], pol);
                else st_stream_v4(dst + i * 16, v[u]);
            }
        }
    }
}

__device__ __forceinline__ void unpack8(const uint4& v, float* a) {
    a[0] = bf16_lo(v.x), a[1] = bf16_hi(v.x), a[2] = bf16_lo(v.y), a[3] = bf16_hi(v.y);
    a[4] = bf16_lo(v.z), a[5] = bf16_hi(v.z), a[6] = bf16_lo(v.w), a[7] = bf16_hi(v.w);
}

// Sum over ranks of one 16-byte vector at byte offset `off` of the symmetric gradient buffer -> fp32 acc[kVec].
template <bool kBf16In, bool kNvls>
__device__ __forceinline__ void reduce_vec(const PeerPtrs& peers, uint64_t mc_base, int rank, int world, int64_t off,
                                           float* acc) {
    constexpr int kVec = kBf16In ? 8 : 4;
    if constexpr (kNvls) {
        unpack8(multimem_ld_reduce_bf16x8(reinterpret_cast<const uint8_t*>(mc_base) + off), acc);
    } else {
#pragma unroll
        for (int q = 0; q < kVec; ++q) acc[q] = 0.f;
        for (int r0 = 0; r0 < world; r0 += 4) {  // 4 peers' loads in flight at a time
            uint4 v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (r0 + j < world) {
                    const int peer = (rank + r0 + j) % world;  // start at self, stagger egress ports
                    v[j] = ld_stream_v4(reinterpret_cast<const uint8_t*>(peers.p[peer]) + off);
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (r0 + j < world) {
                    if constexpr (kBf16In) {
                        float a[8];
                        unpack8(v[j], a);
#pragma unroll
                        for (int q = 0; q < 8; ++q) acc[q] += a[q];
                    } else {
                        acc[0] += __uint_as_float(v[j].x), acc[1] += __uint_as_float(v[j].y);
                        acc[2] += __uint_as_float(v[j].z), acc[3] += __uint_as_float(v[j].w);
                    }
                }
            }
        }
    }
}

// seg_table row (reduce-scatter): [full_off_bytes, shard_off_elems, nelems, chunk_prefix]; chunk = kRsChunkVecs vectors
template <bool kBf16In, bool kNvls, bool kAdam>
__global__ void __launch_bounds__(kCommThreads, kNvls && !kAdam ? 8 : 5)
    reduce_scatter_kernel(PeerPtrs peers, uint64_t mc_base, int rank, int world, SyncArgs sync,
                          float* __restrict__ out, const int64_t* __restrict__ seg, int nseg, int64_t total_chunks,
                          float scale, float* __restrict__ sumsq_out, AdamFuse adam) {
    const uint32_t seq = sync_begin(sync);
    const uint64_t pol = l2_evict_first_policy();
    float sq = 0.f;
    int s = 0;
    constexpr int kVec = kBf16In ? 8 : 4;  // elements per 16 B
    constexpr int kU = kNvls ? kRsUnroll : 1;
    for (int64_t c = blockIdx.x; c < total_chunks; c += gridDim.x) {
        while (s + 1 < nseg && seg[(s + 1) * 4 + 3] <= c) ++s;
        const int64_t* row = seg + s * 4;
        const int64_t v0 = (c - row[3]) * kRsChunkVecs;           // first 16 B vector of this chunk
        const int64_t nvec = min(kRsChunkVecs, row[2] / kVec - v0);
        const int64_t src_off = row[0] + v0 * 16;
        float* dst = out + row[1] + v0 * kVec;
        for (int64_t base = 0; base < nvec; base += kCommThreads * kU) {
            float acc[kU][kVec];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int64_t i = base + threadIdx.x + u * kCommThreads;
                if (i < nvec) reduce_vec<kBf16In, kNvls>(peers, mc_base, rank, world, src_off + i * 16, acc[u]);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int64_t i = base + threadIdx.x + u * kCommThreads;
                if (i >= nvec) continue;
#pragma unroll
                for (int q = 0; q < kVec; ++q) {
                    acc[u][q] *= scale;
                    sq += acc[u][q] * acc[u][q];
                }
                if constexpr (kAdam) {
                    // Sharded AdamW right here: the reduced gradient never goes to memory.
                    const int64_t e = row[1] + (v0 + i) * kVec;  // element offset inside the shard
                    float lr = adam.lr, decay = 1.f - adam.lr * adam.wd;
                    if (adam.groups != nullptr) {  // a vector of kVec elements never crosses a 64-element chunk
                        const int grp = adam.groups[e >> 6];
                        lr = adam.lr * __ldg(adam.group_hyper + 2 * grp);
                        decay = 1.f - lr * __ldg(adam.group_hyper + 2 * grp + 1);
                    }
#pragma unroll
                    for (int q = 0; q < kVec; ++q) {
                        const int32_t bits =
                            (static_cast<int32_t>(adam.hi[e + q]) << 16) + static_cast<int32_t>(adam.lo[e + q]);
                        float w = __int_as_float(bits);
                        const float g = acc[u][q];
                        const float mi = adam.beta1 * adam.m[e + q] + (1.f - adam.beta1) * g;
                        const float vi = adam.beta2 * adam.v[e + q] + (1.f - adam.beta2) * g * g;
                        adam.m[e + q] = mi;
                        adam.v[e + q] = vi;
                        w = w * decay - lr * (mi * adam.inv_bc1) / (sqrtf(vi * adam.inv_bc2) + adam.eps);
                        const int32_t nb = __float_as_int(w);
                        const int32_t h = (nb + 0x8000) >> 16;
                        adam.hi[e + q] = static_cast<uint16_t>(h & 0xFFFF);
                        adam.lo[e + q] = static_cast<int16_t>(nb - (h << 16));
                    }
                } else {
                    uint4 o0, o1;
                    o0.x = __float_as_uint(acc[u][0]), o0.y = __float_as_uint(acc[u][1]);
                    o0.z = __float_as_uint(acc[u][2]), o0.w = __float_as_uint(acc[u][3]);
                    st_stream_v4_hint(dst + i * kVec, o0, pol);
                    if constexpr (kVec == 8) {
                        o1.x = __float_as_uint(acc[u][4]), o1.y = __float_as_uint(acc[u][5]);
                        o1.z = __float_as_uint(acc[u][6]), o1.w = __float_as_uint(acc[u][7]);
                        st_stream_v4_hint(dst + i * kVec + 4, o1, pol);
                    }
                }
            }
        }
    }
    if (sumsq_out != nullptr) {
        sq = warp_sum_f(sq);
        if (threadIdx.x % 32 == 0 && sq != 0.f) atomicAdd(sumsq_out, sq);
    }
    sync_end(sync, seq);
}

// In-place mean over a replicated bf16 buffer that lives at the same symmetric offset on every rank (DDP mode).
// Chunk c (kRsChunkVecs vectors) is reduced by rank c % world and written back to every rank.
template <bool kNvls>
__global__ void __launch_bounds__(kCommThreads, 5)
    all_reduce_kernel(PeerPtrs peers, uint64_t mc_base, SyncArgs sync, int64_t nbytes, float scale) {
    const uint32_t seq = sync_begin(sync);
    const int rank = sync.rank, world = sync.world;
    const int64_t total_vecs = nbytes / 16;
    const int64_t total_chunks = (total_vecs + kRsChunkVecs - 1) / kRsChunkVecs;
    const int64_t my_chunks = (total_chunks - rank + world - 1) / world;
    constexpr int kU = kNvls ? kRsUnroll : 1;
    for (int64_t k = blockIdx.x; k < my_chunks; k += gridDim.x) {
        const int64_t v0 = (k * world + rank) * kRsChunkVecs;
        const int64_t nvec = min(kRsChunkVecs, total_vecs - v0);
        for (int64_t base = 0; base < nvec; base += kCommThreads * kU) {
            float acc[kU][8];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int64_t i = base + threadIdx.x + u * kCommThreads;
                if (i < nvec) reduce_vec<true, kNvls>(peers, mc_base, rank, world, (v0 + i) * 16, acc[u]);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int64_t i = base + threadIdx.x + u * kCommThreads;
                if (i >= nvec) continue;
                uint4 o;
                o.x = pack_bf16x2(acc[u][0] * scale, acc[u][1] * scale);
                o.y = pack_bf16x2(acc[u][2] * scale, acc[u][3] * scale);
                o.z = pack_bf16x2(acc[u][4] * scale, acc[u][5] * scale);
                o.w = pack_bf16x2(acc[u][6] * scale, acc[u][7] * scale);
                const int64_t off = (v0 + i) * 16;
                if constexpr (kNvls) {
                    multimem_st_v4(reinterpret_cast<uint8_t*>(mc_base) + off, o);
                } else {
                    for (int r = 0; r < world; ++r)
                        st_stream_v4(reinterpret_cast<uint8_t*>(peers.p[(rank + r) % world]) + off, o);
                }
            }
        }
    }
    sync_end(sync, seq);
}

// flags layout in every rank's symmetric flag region: uint32 flags[slot][world]
// seq_dev (optional): per-slot sequence counters kept on the device (every rank advances them identically), so
// the same launch can be replayed from a CUDA graph.
__global__ void signal_barrier_kernel(PeerPtrs flag_bases, int rank, int world, int slot, uint32_t seq,
                                      uint32_t* seq_dev) {
    const int r = threadIdx.x;
    if (seq_dev != nullptr) seq = seq_dev[slot] + 1;
    __syncwarp();
    if (r == 0 && seq_dev != nullptr) seq_dev[slot] = seq;
    if (r >= world) return;
    __threadfence_system();
    uint32_t* remote = reinterpret_cast<uint32_t*>(flag_bases.p[r]) + slot * kMaxWorld + rank;
    st_release_sys(remote, seq);
    spin_until(reinterpret_cast<const uint32_t*>(flag_bases.p[rank]) + slot * kMaxWorld + r, seq, rank, r,
               "signal_barrier");
}

// scratch layout in every rank's symmetric region: float scratch[slot][world][kMaxScalars]
constexpr int kMaxScalars = 16;
__global__ void allreduce_scalars_kernel(PeerPtrs flag_bases, PeerPtrs scratch_bases, int rank, int world, int slot,
                                         uint32_t seq, float* __restrict__ vals, int k, int op, uint32_t* seq_dev,
                                         int counter_idx) {
    const int t = threadIdx.x;
    if (seq_dev != nullptr) {  // slot alternates with the parity of the device-side sequence number
        seq = seq_dev[counter_idx] + 1;
        slot = slot + static_cast<int>(seq & 1u);
    }
    __syncthreads();
    if (t == 0 && seq_dev != nullptr) seq_dev[counter_idx] = seq;
    // phase 1: thread (r, j) pushes vals[j] into peer r's scratch[slot][rank][j]
    if (t < world * k) {
        const int r = t / k, j = t % k;
        float* dst = reinterpret_cast<float*>(scratch_bases.p[r]) + (slot * kMaxWorld + rank) * kMaxScalars + j;
        st_relaxed_sys_f32(dst, vals[j]);
    }
    __syncthreads();
    if (t < world) {
        __threadfence_system();
        uint32_t* remote = reinterpret_cast<uint32_t*>(flag_bases.p[t]) + slot * kMaxWorld + rank;
        st_release_sys(remote, seq);
        spin_until(reinterpret_cast<const uint32_t*>(flag_bases.p[rank]) + slot * kMaxWorld + t, seq, rank, t,
                   "allreduce_scalars");
    }
    __syncthreads();
    if (t < k) {
        const float* src = reinterpret_cast<const float*>(scratch_bases.p[rank]) + slot * kMaxWorld * kMaxScalars + t;
        float acc = ld_relaxed_sys_f32(src);
        for (int r = 1; r < world; ++r) {  // fixed order -> bitwise identical on every rank
            const float v = ld_relaxed_sys_f32(src + r * kMaxScalars);
            acc = (op == 0) ? acc + v : fmaxf(acc, v);
        }
        vals[t] = acc;
    }
}

PeerPtrs to_peers(const std::vector<int64_t>& v) {
    if (v.size() > kMaxWorld) throw std::runtime_error("comm: world size > 16 not supported");
    PeerPtrs p;
    for (int i = 0; i < kMaxWorld; ++i) p.p[i] = i < (int)v.size() ? static_cast<uint64_t>(v[i]) : 0;
    return p;
}

inline void check_launch(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

SyncArgs to_sync(const CommSync* cs) {
    SyncArgs s{};
    s.world = 1;
    if (cs != nullptr && cs->world > 1) {
        if (cs->seq_dev == nullptr || cs->cta_ctr == nullptr) throw std::runtime_error("comm: sync needs device counters");
        s.flags = to_peers(cs->flag_ptrs);
        s.rank = cs->rank, s.world = cs->world;
        s.slot_ready = cs->slot_ready, s.slot_done = cs->slot_done;
        s.seq_dev = cs->seq_dev, s.counter_idx = cs->counter_idx, s.cta_ctr = cs->cta_ctr;
    }
    return s;
}

int grid_for(int64_t chunks, int max_ctas) {
    return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(chunks, max_ctas > 0 ? max_ctas : 64)));
}

}  // namespace

void p2p_all_gather(const std::vector<int64_t>& peer_ptrs, int rank, void* out, const int64_t* seg_table_dev,
                    int nseg, int64_t total_chunks, int max_ctas, cudaStream_t stream) {
    (void)rank;
    if (total_chunks == 0) return;
    static const int l2_hint = getenv("B200_COMM_L2_HINT") ? atoi(getenv("B200_COMM_L2_HINT")) : 1;
    p2p_all_gather_kernel<<<grid_for(total_chunks, max_ctas), kCommThreads, 0, stream>>>(
        to_peers(peer_ptrs), static_cast<uint8_t*>(out), seg_table_dev, nseg, total_chunks, l2_hint);
    check_launch("p2p_all_gather");
}

void reduce_scatter(const std::vector<int64_t>& peer_ptrs, int64_t mc_ptr, int rank, int world, float* out,
                    const int64_t* seg_table_dev, int nseg, int64_t total_chunks, bool in_is_bf16, float scale,
                    float* sumsq_out, int max_ctas, cudaStream_t stream, const CommSync* sync, const AdamFuse* adam) {
    if (total_chunks == 0) return;
    const bool nvls = mc_ptr != 0;
    if (nvls && !in_is_bf16) throw std::runtime_error("reduce_scatter: the in-switch reduction path is bf16 only");
    if (adam != nullptr && !in_is_bf16) throw std::runtime_error("reduce_scatter: fused AdamW needs bf16 gradients");
    if (adam != nullptr && (adam->groups == nullptr) != (adam->group_hyper == nullptr))
        throw std::runtime_error("reduce_scatter: the parameter groups need both groups and group_hyper (or neither)");
    const SyncArgs ks = to_sync(sync);  // world <= 1 in there: no flag protocol (caller brackets with barriers)
    const PeerPtrs peers = nvls ? PeerPtrs{} : to_peers(peer_ptrs);
    const uint64_t mc = static_cast<uint64_t>(mc_ptr);
    const AdamFuse a = adam != nullptr ? *adam : AdamFuse{};
    const int grid = grid_for(total_chunks, max_ctas);
#define B200_RS(BF, NV, AD)                                                                                          \
    reduce_scatter_kernel<BF, NV, AD><<<grid, kCommThreads, 0, stream>>>(peers, mc, rank, world, ks, out,             \
                                                                         seg_table_dev, nseg, total_chunks, scale,    \
                                                                         sumsq_out, a)
    if (nvls) {
        if (adam != nullptr) B200_RS(true, true, true);
        else B200_RS(true, true, false);
    } else if (in_is_bf16) {
        if (adam != nullptr) B200_RS(true, false, true);
        else B200_RS(true, false, false);
    } else {
        B200_RS(false, false, false);
    }
#undef B200_RS
    check_launch("reduce_scatter");
}

void all_reduce_mean_bf16(const std::vector<int64_t>& peer_ptrs, int64_t mc_ptr, int rank, int world, int64_t nbytes,
                          float scale, int max_ctas, cudaStream_t stream, const CommSync* sync) {
    if (nbytes == 0 || world <= 1) return;
    if (nbytes % 16 != 0) throw std::runtime_error("all_reduce: buffer size must be a multiple of 16 bytes");
    if (sync == nullptr || sync->world != world) throw std::runtime_error("all_reduce: needs the flag protocol");
    (void)rank;
    const SyncArgs s = to_sync(sync);
    const int64_t chunks = (nbytes / 16 + kRsChunkVecs - 1) / kRsChunkVecs;
    const int grid = grid_for((chunks + world - 1) / world, max_ctas);
    if (mc_ptr != 0)
        all_reduce_kernel<true><<<grid, kCommThreads, 0, stream>>>(PeerPtrs{}, static_cast<uint64_t>(mc_ptr), s, nbytes, scale);
    else
        all_reduce_kernel<false><<<grid, kCommThreads, 0, stream>>>(to_peers(peer_ptrs), 0, s, nbytes, scale);
    check_launch("all_reduce");
}

void signal_barrier(const std::vector<int64_t>& flag_ptrs, int rank, int world, int slot, uint32_t seq,
                    cudaStream_t stream, uint32_t* seq_dev) {
    signal_barrier_kernel<<<1, 32, 0, stream>>>(to_peers(flag_ptrs), rank, world, slot, seq, seq_dev);
    check_launch("signal_barrier");
}

void allreduce_scalars(const std::vector<int64_t>& flag_ptrs, const std::vector<int64_t>& scratch_ptrs, int rank,
                       int world, int slot, uint32_t seq, float* vals, int k, int op, cudaStream_t stream,
                       uint32_t* seq_dev, int counter_idx) {
    if (k > kMaxScalars) throw std::runtime_error("allreduce_scalars: at most 16 values");
    allreduce_scalars_kernel<<<1, 256, 0, stream>>>(to_peers(flag_ptrs), to_peers(scratch_ptrs), rank, world, slot, seq,
                                                   vals, k, op, seq_dev, counter_idx);
    check_launch("allreduce_scalars");
}

int64_t ag_chunk_bytes() { return kAgChunkBytes; }
int64_t rs_chunk_elems() { return kRsChunkElems; }
int64_t rs_chunk_vecs() { return kRsChunkVecs; }
int comm_max_world() { return kMaxWorld; }
int comm_max_scalars() { return kMaxScalars; }

}  // namespace b200
