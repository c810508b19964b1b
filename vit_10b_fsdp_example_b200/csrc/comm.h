// Host API of the NVLink / NVSwitch symmetric-memory collectives (see comm.cu): what XlaFullyShardedDataParallel's
// all_gather / reduce_scatter / all_reduce lower to in the reference (run_vit_training.py:177-181,261-275).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

namespace b200 {

// Segment tables live in device memory (int64).  Row formats:
//   all-gather     : [src_rank, src_off_bytes, dst_off_bytes, nbytes, chunk_prefix]   (chunk = ag_chunk_bytes())
//   reduce-scatter : [full_off_bytes, shard_off_elems, nelems, chunk_prefix]          (chunk = rs_chunk_vecs() 16-byte vectors)
void p2p_all_gather(const std::vector<int64_t>& peer_ptrs, int rank, void* out, const int64_t* seg_table_dev,
                    int nseg, int64_t total_chunks, int max_ctas, cudaStream_t stream);
// Optional AdamW fused into the reduce-scatter epilogue (only legal when gradient clipping is off: the update
// of a shard then needs nothing but its own reduced gradient).  `out` is not written in that case.
struct AdamFuse {
    uint16_t* hi = nullptr;  // split-fp32 master shard (see elementwise.cu)
    int16_t* lo = nullptr;
    float* m = nullptr;
    float* v = nullptr;
    float lr = 0.f, beta1 = 0.9f, beta2 = 0.999f, eps = 1e-8f, wd = 0.f, inv_bc1 = 1.f, inv_bc2 = 1.f;
    // parameter groups (optional): groups[e / 64] is the group of shard element e, group_hyper its fp32 row
    // (lr_scale, wd); the update then uses lr * lr_scale and that wd.  Null = one group (lr, wd).
    const uint8_t* groups = nullptr;
    const float* group_hyper = nullptr;
};
// Cross-GPU flag protocol folded into reduce_scatter / all_reduce (no separate barrier launches): "inputs ready"
// flags are published at kernel start, "done reading" flags by the last CTA, which also waits for every peer's.
// seq_dev[counter_idx] counts the calls (device-resident -> CUDA-graph replayable); cta_ctr is a zeroed device word.
struct CommSync {
    std::vector<int64_t> flag_ptrs;  // every rank's symmetric flag region
    int rank = 0, world = 1;
    int slot_ready = 0, slot_done = 0;
    uint32_t* seq_dev = nullptr;
    int counter_idx = 0;
    uint32_t* cta_ctr = nullptr;
};
// mc_ptr != 0: in-switch reduction (multimem.ld_reduce, bf16 only); otherwise pulls over peer_ptrs.
// sync == nullptr: the caller brackets the call with signal_barrier()s itself.
void reduce_scatter(const std::vector<int64_t>& peer_ptrs, int64_t mc_ptr, int rank, int world, float* out,
                    const int64_t* seg_table_dev, int nseg, int64_t total_chunks, bool in_is_bf16, float scale,
                    float* sumsq_out, int max_ctas, cudaStream_t stream, const CommSync* sync = nullptr,
                    const AdamFuse* adam = nullptr);
// In-place mean over a replicated bf16 buffer at the same symmetric offset on every rank (DDP gradient all-reduce).
void all_reduce_mean_bf16(const std::vector<int64_t>& peer_ptrs, int64_t mc_ptr, int rank, int world, int64_t nbytes,
                          float scale, int max_ctas, cudaStream_t stream, const CommSync* sync);
// flags: uint32 [slot][16] per rank; scratch: float [slot][16][16] per rank (both in symmetric memory)
// seq_dev != nullptr: sequence numbers come from (and are advanced in) device memory -> CUDA-graph replayable.
// For allreduce_scalars the flag/scratch slot is then `slot + (seq & 1)`.
void signal_barrier(const std::vector<int64_t>& flag_ptrs, int rank, int world, int slot, uint32_t seq,
                    cudaStream_t stream, uint32_t* seq_dev = nullptr);
void allreduce_scalars(const std::vector<int64_t>& flag_ptrs, const std::vector<int64_t>& scratch_ptrs, int rank,
                       int world, int slot, uint32_t seq, float* vals, int k, int op, cudaStream_t stream,
                       uint32_t* seq_dev = nullptr, int counter_idx = 0);
int64_t ag_chunk_bytes();
int64_t rs_chunk_elems();
int64_t rs_chunk_vecs();
int comm_max_world();
int comm_max_scalars();

}  // namespace b200
