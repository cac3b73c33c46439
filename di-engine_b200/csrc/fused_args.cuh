#pragma once
// Arguments shared by the two kernels of the one-launch learner step gae -> ppo_error:
// fused.cu (row tiles + cross-CTA chunk counters; also the dispatcher) and colws.cu (column tiles, no cross-CTA dependency).
#include "ppo_math.cuh"

namespace b200rl {

struct FusedArgs {
    PpoArgs p;  // p.adv = the (T*B) advantage buffer this kernel WRITES (phase G) and reads (phase P)
    const float* value;
    float* next_value;
    const float* reward;
    const float* done;
    const float* traj;
    long long T, B;
    float gamma, gl;
    int mask_inplace;
    int defer_wait;  // colws.cu: only the writing warps wait for the previous launches (captured steps, common.cuh)
    int trace;  // colws.cu: per-CTA %globaltimer stamps in the workspace (B200RL_FUSED_TRACE=1; tools/trace_col.py)
    // optional data-parallel exchange of the six loss scalars, fused into the step's finalize launch (colws.cu; common.cuh)
    const unsigned long long* x_mailboxes;
    unsigned int* x_seq;
    float* x_out_mean;
    int x_rank, x_world;
};

// colws.cu: column tiles, warp-specialised (loader / scanner / consumer warps, mbarrier pipeline, cp.async copies).
// colws_ok: the shapes, 16-byte alignment and the ring of at least two stages at two CTAs per SM the kernel needs.
bool colws_ok(const FusedArgs& f);
int launch_colws(const FusedArgs& f, bool grads, float* out, float* ws, size_t ws_bytes, cudaStream_t st);

}  // namespace b200rl
