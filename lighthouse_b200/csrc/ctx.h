// ctx.h — process-wide library context: one process drives one GPU (one rank per GPU).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/lhb200.h"

namespace lhb200 {

struct Ctx {
    bool ready = false;
    int device = -1;
    cudaStream_t stream = nullptr;
    std::recursive_mutex mu;  // host entry points are serialised (callers are spawn_blocking workers)
    std::atomic<uint64_t> launches{0};
    uint8_t zero_hashes[65][32];
    // scratch for host-buffer entry points
    void* d_scratch = nullptr;
    size_t d_scratch_bytes = 0;
    void* h_pinned = nullptr;
    size_t h_pinned_bytes = 0;
};

Ctx& ctx();
void set_error(const char* fmt, ...);
int32_t cuda_fail(cudaError_t e, const char* what);
// grow-only scratch (device / pinned host); returns nullptr on failure (error set)
void* dev_scratch(size_t nbytes);
void* pinned_scratch(size_t nbytes);

#define LHB_CUDA(expr)                                                 \
    do {                                                               \
        cudaError_t _e = (expr);                                       \
        if (_e != cudaSuccess) return ::lhb200::cuda_fail(_e, #expr);  \
    } while (0)

#define LHB_REQUIRE_READY()                                                          \
    do {                                                                             \
        if (!::lhb200::ctx().ready) {                                                \
            ::lhb200::set_error("lhb200_init() has not succeeded (no CPU fallback)"); \
            return LHB200_ENODEV;                                                    \
        }                                                                            \
    } while (0)

// the library's NCCL communicator (comm.cu); no-ops / local copies when no communicator is initialised
bool comm_active();
int comm_world();
int comm_rank();
int32_t comm_allreduce_min_u8(void* d_buf, size_t n, cudaStream_t s);
int32_t comm_allgather_bytes(const void* d_send, void* d_recv, size_t bytes_per_rank, cudaStream_t s);

inline void count_launch(uint64_t n = 1) { ctx().launches.fetch_add(n, std::memory_order_relaxed); }

// A pooled BLS batch handle driven from outside bls_host.cu (lhb200_attestations_verify): borrow, keep scratch on it,
// stage sets whose key indices the caller writes on the device, verify, return.  No library mutex is held.
lhb200_bls_batch* bls_pool_borrow(uint32_t n_sets);
void bls_pool_return(lhb200_bls_batch* b);
cudaStream_t bls_batch_stream(const lhb200_bls_batch* b);
void* bls_batch_aux(lhb200_bls_batch* b, size_t dev_bytes, uint8_t** pinned, size_t pinned_bytes);
int32_t bls_batch_stage_table(lhb200_bls_batch* b, const lhb200_pubkey_table* table, const uint8_t* sigs,
                              const uint8_t* msgs, const uint32_t* pk_offsets, const uint64_t* rands, uint32_t n_sets,
                              uint32_t** d_key_indices);
int32_t bls_batch_finish(lhb200_bls_batch* b, uint8_t* ok, uint8_t* set_status);
int32_t bls_batch_local_keys(lhb200_bls_batch* b, const uint8_t* d_pk48, uint32_t n, uint8_t* d_status);
uint64_t bls_last_batch_launches();   // launches of the calling thread's last bls_batch_finish (0: none)

}  // namespace lhb200
