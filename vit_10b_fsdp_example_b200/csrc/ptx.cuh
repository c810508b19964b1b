// Thin inline-PTX wrappers for the Hopper (sm_90a) execution model:
// mbarrier, TMA (cp.async.bulk.tensor), cluster helpers, register reallocation and small packing helpers.
// The wgmma wrappers live in wgmma.cuh.
//
// Everything here is hand-written PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>

namespace b200 {

#ifndef B200_SPIN_LIMIT
// Bounded spin: a stuck barrier traps (-> launch error) instead of hanging the GPU.
// ~2^31 polls of a try_wait with a HW suspend-time hint is many seconds.
#define B200_SPIN_LIMIT (1u << 28)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() {
    uint32_t l;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
    return l;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "elect.sync _|P1, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void cluster_arrive() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait() {
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_sync() {
    cluster_arrive();
    cluster_wait();
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Arrive on the barrier at the same smem offset in CTA `cta` of this cluster.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    asm volatile(
        "{\n\t"
        ".reg .b32 raddr;\n\t"
        "mapa.shared::cluster.u32 raddr, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [raddr];\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(cta)
        : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t phase) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
    return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, phase)) {
        if (++spins > B200_SPIN_LIMIT) {
            printf("[b200] mbarrier timeout: block %d thread %d bar %u phase %u\n", blockIdx.x, threadIdx.x,
                   smem_u32(bar), phase);
            __trap();
        }
    }
}

// The same bounded wait without the diagnostic printf, for kernels that issue wgmma: a printf is a function call, and
// any call in such a kernel makes ptxas serialise every wgmma (warning C7510: each MMA waits for the previous one).
__device__ __forceinline__ void mbar_wait_silent(uint64_t* bar, uint32_t phase) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, phase)) {
        if (++spins > B200_SPIN_LIMIT) __trap();
    }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// 4-D tiled load, 1-CTA flavour. Completion on `bar` (in this CTA).
__device__ __forceinline__ void tma_load_4d(const void* tmap, uint64_t* bar, void* smem, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// 4-D tiled load multicast to every CTA of the cluster in `cta_mask`: the box lands at the same smem offset in each
// of them and completes bytes on the mbarrier at `bar`'s offset in each of them.
__device__ __forceinline__ void tma_load_4d_multicast(const void* tmap, uint64_t* bar, void* smem, int c0, int c1,
                                                      int c2, int c3, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(smem)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"(cta_mask)
        : "memory");
}

__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* smem, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
            reinterpret_cast<uint64_t>(tmap)),
        "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }

template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// Register reallocation between the producer and the consumer warpgroups
// ----------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ void reg_dealloc() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void reg_alloc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------------------------
// Misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t a) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(a) : "memory");
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

}  // namespace b200
