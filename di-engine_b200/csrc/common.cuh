// Shared device helpers for the b200rl kernels (sm_90a, H100).
//
// Conventions used by every kernel in this directory
//   * trajectory tensors are row-major (T, C): time is the slow axis, the batch "column" c is contiguous, so a
//     warp reads 128 contiguous bytes of one time-step and a CTA owns a tile of columns for all T;
//   * loss heads reduce warp -> CTA -> grid inside the same kernel: every CTA stores its partial sums to the
//     caller-provided workspace and the last CTA to arrive (ticket from one atomic) adds them up in a fixed
//     order in fp64 -- deterministic, no second launch, no host sync;
//   * expressions whose rounding must match the reference's separate torch ops use __fmul_rn/__fadd_rn so ptxas
//     cannot contract them into FMAs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#define B200RL_OK 0
#ifndef B200RL_ERR_ARG
#define B200RL_ERR_ARG (-1)
#define B200RL_ERR_WORKSPACE (-2)
#endif

// workspace layout (floats): [0,16) control words, [16, ...) per-CTA partial sums
#define WS_CTRL_WORDS 16
#define WS_MIN_BYTES (1u << 20)

namespace b200rl {

// SMs of an H100 SXM: grid-stride caps and the SM-count-derived tile-width thresholds are multiples of it.  Kernels whose
// grid must match residency exactly query cudaDevAttrMultiProcessorCount instead, so on a GPU with another SM count (an
// H100 PCIe has 114) only these heuristics are off, never correctness.
constexpr int NUM_SMS = 132;

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }

// streaming loads / stores: every tensor on this path is touched once per launch
__device__ __forceinline__ float ldg_stream(const float* p) { return __ldcs(p); }
__device__ __forceinline__ float4 ldg_stream4(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ void stg_stream(float* p, float v) { __stcs(p, v); }
__device__ __forceinline__ void stg_stream4(float4* p, float4 v) { __stcs(p, v); }

// release/acquire fence at GPU scope (MEMBAR.ALL.GPU) -- what the "write results, then signal a counter" patterns of this
// library need; __threadfence() is the sequentially-consistent flavour (MEMBAR.SC.GPU), measurably slower under load
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Grid-wide sum of K per-thread partials.  After the call, in the LAST CTA to finish (returns true there, false
// elsewhere) thread 0 holds the grid totals in tot[0..K).  `ws` must hold WS_CTRL_WORDS + gridDim.x*K floats,
// control word `slot` must be zero on entry and is reset to zero on exit (stream-ordered reuse).
template <int K, int NT>
__device__ __forceinline__ bool grid_sum(float (&v)[K], double (&tot)[K], float* ws, int slot) {
    __shared__ float s_part[K][NT / 32];
    __shared__ double s_tot[K][NT / 32];
    __shared__ bool s_last;
    __shared__ volatile unsigned int s_dep;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float r = warp_sum(v[k]);
        if (lane == 0) s_part[k][wid] = r;
    }
    __syncthreads();
    float* part = ws + WS_CTRL_WORDS;
    unsigned int* ctrl = reinterpret_cast<unsigned int*>(ws);
    if (threadIdx.x == 0) {
        // Publish this CTA's partial sums with RETURNING atomics (performed at L2, so they are visible device-wide once
        // they return) and make the ticket depend on their return values.  This replaces "plain stores + gpu-scope
        // fence + ticket": the fence had to wait for every outstanding store of the SM (the gradient tiles of the fused
        // kernels), which put that drain on the critical path of the grid reduction.
        unsigned int dep = 0u;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            float r = 0.f;
#pragma unroll
            for (int w = 0; w < NT / 32; ++w) r += s_part[k][w];
            dep |= atomicExch(reinterpret_cast<unsigned int*>(&part[(size_t)blockIdx.x * K + k]), __float_as_uint(r));
        }
        s_dep = dep;  // a real use of the returned values: instructions issue in order, so everything below waits here
        asm volatile("" ::: "memory");
        // release: the partials above (and, through the barrier before, whatever the CTA's threads stored) happen-before
        // the ticket; acquire: the last CTA's reads below happen-after every earlier ticket (PTX memory model, gpu scope)
        unsigned int ticket;
        asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(&ctrl[slot]) : "memory");
        s_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return false;
    fence_acq_rel_gpu();  // every thread of the last CTA reads other CTAs' results: order those reads after the ticket
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] = 0.0;
    // fixed summation order (deterministic); U rows of partials are loaded before any is consumed so the L2 latency of
    // this serial tail is paid once, not once per row
    constexpr int U = 8;
    for (unsigned int b0 = threadIdx.x; b0 < gridDim.x; b0 += NT * U) {
        float v_[U][K];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const unsigned int b = b0 + u * NT;
#pragma unroll
            for (int k = 0; k < K; ++k) v_[u][k] = (b < gridDim.x) ? __ldcg(&part[(size_t)b * K + k]) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
            for (int k = 0; k < K; ++k) acc[k] += (double)v_[u][k];
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double r = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        if (lane == 0) s_tot[k][wid] = r;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double r = 0.0;
#pragma unroll
            for (int w = 0; w < NT / 32; ++w) r += s_tot[k][w];
            tot[k] = r;
        }
        ctrl[slot] = 0u;
    }
    return true;
}

// Grid reduction with ONE atomic round trip per CTA for the SMALL, latency-bound kernels (q-n-step, C51, ...): no ticket, no
// fence, no second read -- and nothing that relies on when another CTA's plain stores become visible.
// Every sum k owns two packed 64-bit accumulators in the workspace.  A CTA turns its partial sum (double) into 128-bit fixed
// point c = hi + lo*2^-40 and adds   word0 += lo<<9 | 1,   word1 += hi<<18 | spill<<9 | 1   with two returning atomics in
// flight together.  The low 9 bits count the CTAs that have added (grid <= 511): the CTA whose add to word0 returns
// count == grid-1 knows that word0 is complete and equal to (returned + own); it takes word1 the same way (or, if another
// CTA's add to word1 is still in flight, polls it until its count is complete), calls fin(k, total) and resets both words for
// the next launch.  Integer addition is associative: the result is bit-identical from run to run whatever the order of
// arrival.  Resolution 2^-40 absolute for |CTA partial| < 2^36.  A CTA whose partial is larger or not finite ("spilled")
// counts itself in word1's spill field and first adds, to two more words of sum k,
//   word2 += m2<<9 | 1,   word3 += m3<<36 | nan<<27 | -inf<<18 | +inf<<9 | 1
// where c = m3*2^81 + m2*2^36 + rest exactly, every part with c's sign (|m2| < 2^45 and |m3| < 2^18 signed fields,
// |rest| < 2^36 goes to words 0 / 1 as usual);
// a non-finite partial, or a finite one of 2^99 or more, adds rest = 0 and counts as NaN / -inf / +inf.  The last CTA
// polls words 2 and 3 until their counts equal the spill count, so the total is the exact fixed-point sum for every finite
// partial below 2^99 (6.3e29), +-inf / NaN as the rows give it, and bit-identical from run to run.  A launch without a
// spilled CTA never touches words 2 / 3.  A one-CTA grid skips the atomics.  (In the big streaming kernels the same scheme
// LOSES to a dependent finalize launch -- the atomics return only after the SM's store traffic has drained.)
#define WS_FX_OFF_WORDS 257024   // 16 packed u64 accumulators (zero between launches), above every kernel's partial sums
#define WS_FX_SPILL_WORDS 257088 // 16 more (words 2 / 3 of each sum), past the statistics ticket policy.cu keeps at +48
constexpr int FX_MAX_K = 8;
constexpr unsigned int FX_MAX_GRID = 511;

__device__ __forceinline__ unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// A spilled CTA partial c (|c| >= 2^36 or not finite): adds its words 2 / 3 (a2 points at them) and returns the rest for
// words 0 / 1.  Every step is exact: c / 2^81 and c / 2^36 are power-of-two scalings, and the quotients are truncated
// toward zero, so each m*2^k has c's sign and at most c's magnitude, and c - m*2^k is a multiple of c's last bit smaller
// than c (flooring instead would turn a negative c into 2^81 - |c| and round its low bits away).
static __device__ __noinline__ double fx_spill(double c, unsigned long long* a2) {
    long long m2 = 0;
    unsigned long long w3 = 1ull;
    double rest = 0.0;
    if (c != c) {
        w3 += 1ull << 27;
    } else if (!(fabs(c) < 633825300114114700748351602688.0)) {  // 2^99, and +-inf
        w3 += c > 0.0 ? (1ull << 9) : (1ull << 18);
    } else {
        const double m3 = trunc(c * (1.0 / 2417851639229258349412352.0));  // 2^81
        const double r3 = c - m3 * 2417851639229258349412352.0;
        const double f2 = trunc(r3 * (1.0 / 68719476736.0));               // 2^36
        rest = r3 - f2 * 68719476736.0;
        m2 = (long long)f2;
        w3 += (unsigned long long)(long long)m3 << 36;
    }
    atomicAdd(a2, ((unsigned long long)m2 << 9) + 1ull);
    atomicAdd(a2 + 1, w3);
    return rest;
}

// The last CTA of a launch with `spilled` spilled CTAs: waits for their words 2 / 3, resets them and adds them to the total
// of words 0 / 1.
static __device__ __noinline__ double fx_spill_total(double tot, unsigned long long* a2, unsigned int spilled) {
    unsigned long long t2, t3;
    do t2 = ld_relaxed_gpu_u64(a2); while ((unsigned int)(t2 & 511ull) != spilled);
    do t3 = ld_relaxed_gpu_u64(a2 + 1); while ((unsigned int)(t3 & 511ull) != spilled);
    a2[0] = 0ull;
    a2[1] = 0ull;
    const unsigned int pinf = (unsigned int)(t3 >> 9) & 511u, ninf = (unsigned int)(t3 >> 18) & 511u,
                       nan = (unsigned int)(t3 >> 27) & 511u;
    if (nan || (pinf && ninf)) return (double)__int_as_float(0x7fc00000);
    if (pinf) return (double)INFINITY;
    if (ninf) return -(double)INFINITY;
    return tot + (double)((long long)t2 >> 9) * 68719476736.0 + (double)((long long)t3 >> 36) * 2417851639229258349412352.0;
}

template <int K, int NT, class Fin>
__device__ __forceinline__ void grid_sum_fx(float (&v)[K], float* ws, Fin fin) {
    static_assert(K <= FX_MAX_K, "K");
    __shared__ float s_fx[K][NT / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float r = warp_sum(v[k]);
        if (lane == 0) s_fx[k][wid] = r;
    }
    __syncthreads();
    if (threadIdx.x >= K) return;
    const int k = threadIdx.x;
    double c = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) c += (double)s_fx[k][w];
    if (gridDim.x == 1) {
        fin(k, c);
        return;
    }
    const bool bad = !(fabs(c) < 68719476736.0);  // 2^36; also catches NaN
    unsigned long long* a2 = reinterpret_cast<unsigned long long*>(ws + WS_FX_SPILL_WORDS) + 2 * k;
    long long hi = 0;
    unsigned long long lo = 0;
    if (!bad) {
        const double fl = floor(c);
        hi = (long long)fl;
        lo = (unsigned long long)((c - fl) * 1099511627776.0);  // (c - floor c) is exact; 2^40
    } else {
        const double r = fx_spill(c, a2);  // |r| < 2^36
        const double fl = floor(r);
        hi = (long long)fl;
        lo = (unsigned long long)((r - fl) * 1099511627776.0);
    }
    const unsigned long long w0 = (lo << 9) + 1ull;
    const unsigned long long w1 = ((unsigned long long)hi << 18) + (bad ? (1ull << 9) : 0ull) + 1ull;
    unsigned long long* a0 = reinterpret_cast<unsigned long long*>(ws + WS_FX_OFF_WORDS) + 2 * k;
    const unsigned long long old0 = atomicAdd(a0, w0);
    const unsigned long long old1 = atomicAdd(a0 + 1, w1);
    if ((unsigned int)(old0 & 511ull) != gridDim.x - 1) return;
    const unsigned long long t0 = old0 + w0;
    unsigned long long t1 = old1 + w1;
    while ((unsigned int)(t1 & 511ull) != gridDim.x) t1 = ld_relaxed_gpu_u64(a0 + 1);
    const unsigned int spilled = (unsigned int)(t1 >> 9) & 511u;
    const double tot = (double)((long long)t1 >> 18) + (double)(t0 >> 9) * (1.0 / 1099511627776.0);
    a0[0] = 0ull;  // every CTA of this launch has added; the next launch adds only after this one has completed
    a0[1] = 0ull;
    fin(k, spilled ? fx_spill_total(tot, a2, spilled) : tot);
}

// Two-launch variant of the grid reduction for the big streaming kernels: every CTA just stores its K partial sums (no
// atomics, no fence, no ticket -- kernel completion publishes them) and finalize_sums_kernel, a single small CTA launched
// right behind, adds them in a fixed order (deterministic), scales, writes the results and clears `n_clear` control
// words.  The in-kernel ticket path would give the big kernels a serial tail (the partial publication becomes visible only
// behind the SM's outstanding traffic, then the last CTA adds); a dependent tiny launch costs less.
template <int K, int NT>
__device__ __forceinline__ void grid_store_partials(float (&v)[K], float* ws) {
    __shared__ float s_part2[K][NT / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float r = warp_sum(v[k]);
        if (lane == 0) s_part2[k][wid] = r;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        float r = 0.f;
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) r += s_part2[threadIdx.x][w];
        ws[WS_CTRL_WORDS + (size_t)blockIdx.x * K + threadIdx.x] = r;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Data-parallel exchange of the loss scalars without a launch of its own and without anything on the critical path
// (SURVEY section 8e: mean of the rank means, ding/utils/pytorch_ddp_dist_helper.py:38-47), software-pipelined over the
// launches the learner step makes anyway:
//   finalize_sums of step q      (thread k, after writing out[k])   stages {tag q, out[k]} in LOCAL memory -- two plain stores;
//   streaming kernel of step q+1 (first CTA, consumer warp k, while it waits for its first chunk to land anyway)
//                                 consumes the entries tagged q-1 of all ranks from its own mailbox into out_mean[k] (they
//                                 were published a whole step ago), then publishes the staged {q, value} as ONE 8-byte store
//                                 into every peer's mailbox (peer-mapped symmetric memory over NVLink).
// Both the remote stores (complete only when their acknowledgement has crossed NVLink) and the system-scope reads of the
// mailbox are hidden behind the time the kernel streams; in the short finalize launch they would sit on the critical path
// of every step.  Value and tag travel in a single store,
// so no flag ordering is needed.  Two mailbox slots alternate by tag parity; warp k consumes tag q-1 BEFORE it publishes tag q,
// so when a rank publishes tag q+1 (same slot as q-1) every peer's tag q has arrived, i.e. every peer has consumed q-1.
// out_mean[k] is the mean of the latest consumed step (two steps behind out[k]), out_mean[8+k] the one before;
// b200rl_p2p_drain_mean after the last step publishes / consumes the tail so that out_mean[k] is the LAST step's mean.
//
// (Not used: summing the partials INSIDE the streaming kernel with one returning atomic round trip per CTA on packed
// fixed-point accumulators -- bit-reproducible and one launch fewer, but the atomics return only after the SM's store
// traffic has drained, which lengthens the kernel by more than the launch it saves.)
// ---------------------------------------------------------------------------------------------------------------
#define WS_PARTIAL_LIMIT_WORDS 256000  // per-CTA partial sums of every kernel stay below this word of the workspace
constexpr int P2P_SLOT_VALS = 8;       // u64 entries per (slot, rank) in an exchange mailbox

struct XchgArgs {
    const unsigned long long* mailboxes;  // nullable: device array [world] of mailbox base addresses as seen from this rank
    unsigned int* state;                  // 24 words owned by the exchange (zero-initialised): [0,8) staged tags, [8,16) staged
                                          // values, [16,24) last consumed tags
    float* out_mean;                      // 16 floats: [0,8) mean over ranks of the latest consumed step, [8,16) the one before
    int rank, world;
};

__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// finalize launch, thread k, after it has produced res = out[k]: stage this step's value (local stores only)
__device__ __forceinline__ void p2p_stage(const XchgArgs& x, int k, float res) {
    x.state[8 + k] = __float_as_uint(res);
    x.state[k] = x.state[k] + 1u;  // only the thread that owns value k writes state[k] / state[8 + k]
}

// one warp per value k (all 32 lanes call; world <= 32): consume the entries tagged `q` of all ranks -- lane r polls rank r's
// entry, lane 0 adds them in rank order (deterministic) -- and shift out_mean
__device__ __forceinline__ void p2p_consume_warp(const XchgArgs& x, int k, unsigned int q) {
    const int lane = threadIdx.x & 31;
    float v = 0.f;
    if (lane < x.world) {
        const unsigned long long* e = reinterpret_cast<const unsigned long long*>(x.mailboxes[x.rank]) +
                                      ((size_t)(q & 1u) * x.world + lane) * P2P_SLOT_VALS + k;
        unsigned long long w;
        while ((unsigned int)((w = ld_relaxed_sys_u64(e)) >> 32) != q) __nanosleep(32);
        v = __uint_as_float((unsigned int)w);
    }
    float acc = 0.f;
    for (int r = 0; r < x.world; ++r) acc += __shfl_sync(0xffffffffu, v, r);
    if (lane == 0) {
        x.out_mean[8 + k] = x.out_mean[k];
        x.out_mean[k] = acc / (float)x.world;
        x.state[16 + k] = q;
    }
    __syncwarp();
}

// one warp per value k: lane p publishes the staged {tag, value} to rank p's mailbox
__device__ __forceinline__ void p2p_publish_warp(const XchgArgs& x, int k) {
    const int lane = threadIdx.x & 31;
    const unsigned int q = x.state[k];
    if (q == 0u || lane >= x.world) return;
    const unsigned long long word = ((unsigned long long)q << 32) | (unsigned long long)x.state[8 + k];
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(x.mailboxes[lane]) +
                              ((size_t)(q & 1u) * x.world + x.rank) * P2P_SLOT_VALS + k;
    st_relaxed_sys_u64(dst, word);
}

// prologue of the long kernel of step q+1, warp k of its first CTA: consume tag q-1, then publish tag q
__device__ __forceinline__ void p2p_pipeline_warp(const XchgArgs& x, int k) {
    const unsigned int q = x.state[k];
    if (q >= 2u && x.state[16 + k] < q - 1u) p2p_consume_warp(x, k, q - 1u);  // (not again after a drain)
    __syncwarp();
    p2p_publish_warp(x, k);
}

struct FinalizeArgs {
    double scale[8];     // out[k] = sum_k * scale[k]
    int k;               // number of sums
    int n_blocks;        // partial rows
    int clear_ctrl_from, clear_ctrl_n;  // control words [from, from+n) to zero
    int clear_tail_off, clear_tail_n;   // workspace words [off, off+n) to zero (scheduling counters)
    XchgArgs x;                         // optional data-parallel exchange of the K results (x.mailboxes != null)
};

static __global__ void __launch_bounds__(256) finalize_sums_kernel(const float* __restrict__ ws, float* __restrict__ out,
                                                            float* __restrict__ ws_rw, FinalizeArgs fa) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    __shared__ double s_acc[8][8];
    const int K = fa.k;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.0;
    const float* part = ws + WS_CTRL_WORDS;
    for (int b = threadIdx.x; b < fa.n_blocks; b += 256) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < K) acc[k] += (double)part[(size_t)b * K + k];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        double r = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        if (lane == 0) s_acc[k][wid] = r;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        double r = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) r += s_acc[threadIdx.x][w];
        const float res = (float)(r * fa.scale[threadIdx.x]);
        out[threadIdx.x] = res;
        if (fa.x.mailboxes) p2p_stage(fa.x, threadIdx.x, res);  // data-parallel exchange: the next step's kernel publishes it
    }
    unsigned int* wsu = reinterpret_cast<unsigned int*>(ws_rw);
    for (int i = threadIdx.x; i < fa.clear_ctrl_n; i += 256) wsu[fa.clear_ctrl_from + i] = 0u;
    for (int i = threadIdx.x; i < fa.clear_tail_n; i += 256) wsu[fa.clear_tail_off + i] = 0u;
}

// log-softmax statistics of one row of n logits read through `ld(j)`; L cooperating lanes (1 or 32) stride the row.
// Returns lse = logsumexp(z) and entropy H = -sum_j p_j log p_j with p_j = exp(z_j - lse)  (torch Categorical:
// logits - logsumexp, entropy = -(logits * softmax).sum(-1)).
template <int L, class Ld>
__device__ __forceinline__ void row_lse_entropy(Ld ld, int n, int lane, float& lse, float& ent) {
    float m = -INFINITY;
    for (int j = lane; j < n; j += L) m = fmaxf(m, ld(j));
    if (L == 32) m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < n; j += L) s += expf(ld(j) - m);
    if (L == 32) s = warp_sum(s);
    lse = m + logf(s);
    float h = 0.f;
    for (int j = lane; j < n; j += L) {
        float lp = ld(j) - lse;
        h += expf(lp) * fmaxf(lp, -3.402823466e38f);
    }
    if (L == 32) h = warp_sum(h);
    ent = -h;
}

template <int L, class Ld>
__device__ __forceinline__ float row_lse(Ld ld, int n, int lane) {
    float m = -INFINITY;
    for (int j = lane; j < n; j += L) m = fmaxf(m, ld(j));
    if (L == 32) m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < n; j += L) s += expf(ld(j) - m);
    if (L == 32) s = warp_sum(s);
    return m + logf(s);
}

// ---------------------------------------------------------------------------------------------------------------
// TMA 1-D bulk copies (cp.async.bulk -> SASS UBLKCP) completing on an mbarrier, and bulk stores tracked by bulk groups.
// Addresses and sizes must be multiples of 16 bytes.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// make generic-proxy shared-memory writes visible to the async proxy (TMA store source)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------------
// 16-byte cp.async (LDGSTS) copies: per-thread groups, or completion counted on an mbarrier
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cpa16(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// same with the shared-memory address already converted (loops that step it by a constant)
__device__ __forceinline__ void cpa16_s(uint32_t smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
// Loader-warp copy of R row segments of P = PG * G 16-byte pieces each: `rstride` bytes apart in global memory, packed in shared
// memory.  lane -> (piece o of every G-piece group, row r of every 32/G-row pass): ONE address computation per lane, every copy
// at an immediate offset from it -- the flat p -> (row, piece) loop it replaces spent ~35 instructions per copy on the division
// and the 64-bit row * stride product, and the loader warp is the longest serial chain of a chunk.
// Requires full rows (no ragged tile / chunk): the callers keep the flat loop for those.
template <int G, int R, int PG>  // PG = 0: runtime `pg_rt`
__device__ __forceinline__ void warp_copy_rows(uint32_t dst, const void* src, long long rstride, int pg_rt, int lane) {
    constexpr int RP = 32 / G;
    static_assert(R % RP == 0, "rows per pass");
    const int o = lane & (G - 1), r = lane / G;
    const int pg = PG ? PG : pg_rt;
    const unsigned char* s = reinterpret_cast<const unsigned char*>(src) + r * rstride + o * 16;
    uint32_t d = dst + (uint32_t)(r * pg * G + o) * 16u;
#pragma unroll
    for (int pass = 0; pass < R / RP; ++pass) {
#pragma unroll
        for (int k = 0; k < pg; ++k) cpa16_s(d + (uint32_t)k * (G * 16u), s + (size_t)k * (G * 16));
        s += RP * rstride;
        d += (uint32_t)(RP * pg * G) * 16u;
    }
}
__device__ __forceinline__ void cpa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cpa_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// arrive on `bar` once all cp.async issued so far by this thread have landed (counts against the barrier's init count)
__device__ __forceinline__ void cpa_mbar_arrive(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Every kernel of this library starts with pdl_prologue(): it lets the NEXT
// kernel in the stream begin launching right away (its launch latency and prologue overlap this kernel's execution) and
// then waits until all PREVIOUS kernels in the stream have completed and flushed their results -- so the usual stream
// ordering of memory is preserved while the launch gap between dependent kernels disappears.
// Host side: launch_k() sets cudaLaunchAttributeProgrammaticStreamSerialization (B200RL_PDL=0 disables it) and returns
// the launch's own error; an operator returns the error of the first launch that fails and queues nothing after it.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_prologue() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

static inline bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("B200RL_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

// B200RL_FUSED_TRACE=1: the column-tile kernels of colws.cu and vtws.cu store per-CTA %globaltimer stamps in the
// workspace (tools/trace_col.py)
static inline bool trace_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("B200RL_FUSED_TRACE");
        v = (e && e[0] == '1') ? 1 : 0;
    }
    return v == 1;
}

// A failed runtime call also records its error as the thread's last error: clear it, so that the library leaves no
// error pending for an unrelated later call to pick up, and return it.
static inline int cuda_rc(cudaError_t e) {
    if (e != cudaSuccess) (void)cudaGetLastError();
    return (int)e;
}

template <typename... KArgs, typename... Args>
static inline int launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cuda_rc(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
}

static inline int launch_finalize(float* ws, float* out, const FinalizeArgs& fa, cudaStream_t st) {
    return launch_k(finalize_sums_kernel, 1, 256, 0, st, (const float*)ws, out, ws, fa);
}

// finalize of the six PPO loss sums (policy, value, entropy, kl, approx_kl, clipfrac) over S samples; the kl sum counts
// only with pretrained logits
static inline FinalizeArgs ppo_finalize_args(long long S, bool has_pre, int grid) {
    FinalizeArgs fa{};
    const double is = 1.0 / (double)S;
    fa.scale[0] = is; fa.scale[1] = 0.5 * is; fa.scale[2] = is; fa.scale[3] = has_pre ? is : 0.0;
    fa.scale[4] = is; fa.scale[5] = is;
    fa.k = 6; fa.n_blocks = grid;
    return fa;
}

// finalize of the three V-trace loss sums (policy, value, entropy) over T*B transitions
static inline FinalizeArgs vtrace_finalize_args(long long T, long long B, int grid) {
    FinalizeArgs fa{};
    const double im = 1.0 / ((double)T * (double)B);
    fa.scale[0] = -im; fa.scale[1] = im; fa.scale[2] = im;
    fa.k = 3; fa.n_blocks = grid;
    return fa;
}

// ---------------------------------------------------------------------------------------------------------------
// Forward-written gradients (include/b200rl.h states the contract).  The forward launch of a loss also writes its gradients
// for the upstream gradients the call site expects and records the values it used; the backward ("verify") launch of the
// same loss returns at once when the actual upstream gradients are bit-identical to that record, and recomputes otherwise.
// Slot k of every record: 0 policy, 1 value, 2 entropy, 3 kl; `owned` is the mask of the slots a kernel computes.
// ---------------------------------------------------------------------------------------------------------------
struct UpstreamRecord {
    const float* g[4];  // the upstream gradients the launch applies, device scalars (nullable = 0): forward the expected,
                        // verify the actual ones
    float* used;        // forward: receives every slot (nullable); verify: compared (null = recompute)
    float* hint;        // verify: its owned slots are refreshed with the actual values (nullable)
    int verify;         // which of the two launches this is
};

// the record of a forward launch: `expected` holds one device float per slot (nullable = 0)
static inline UpstreamRecord forward_record(const float* expected, float* used) {
    UpstreamRecord r{};
    for (int k = 0; k < 4; ++k) r.g[k] = expected ? expected + k : nullptr;
    r.used = used;
    return r;
}

// the record of a verify launch: the actual upstream gradient of every slot
static inline UpstreamRecord verify_record(const float* g0, const float* g1, const float* g2, const float* g3,
                                           const float* used, float* hint) {
    return UpstreamRecord{{g0, g1, g2, g3}, const_cast<float*>(used), hint, 1};
}

// the upstream gradient of slot k, 0 for a slot the kernel does not own
__device__ __forceinline__ float upstream_value(const UpstreamRecord& r, unsigned owned, int k) {
    return ((owned >> k) & 1u) && r.g[k] ? *r.g[k] : 0.f;
}

// g[k] = upstream_value of every slot.  Block 0, thread 0 records every slot in `used` (forward; an unowned one as 0) or
// refreshes the owned slots in `hint` (verify).  -> true when the verify launch may return: `used` is given and every owned
// slot of it is bit-identical to the actual value -- the same decision in every thread of the grid.  `verify` is r.verify,
// or a constant where the kernel's mode is a template parameter (the compiler then drops the other mode's code).  Every
// load comes before the one store, so the loads are issued together: a verify launch that returns at once sits between
// two steps of the training loop.
template <int K>
__device__ __forceinline__ bool upstream(const UpstreamRecord& r, bool verify, unsigned owned, float (&g)[K]) {
    const bool cmp = verify && r.used != nullptr;
    bool same = cmp;
#pragma unroll
    for (int k = 0; k < K; ++k) g[k] = upstream_value(r, owned, k);
#pragma unroll
    for (int k = 0; k < K; ++k)
        if (cmp && ((owned >> k) & 1u)) same &= __float_as_uint(g[k]) == __float_as_uint(r.used[k]);
    float* rec = verify ? r.hint : r.used;
    if (rec && blockIdx.x == 0 && threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < K; ++k)
            if (!verify || ((owned >> k) & 1u)) rec[k] = g[k];
    return same;
}

// The argument rule of every entry point with a record.  verify: the launch may have to recompute, so it needs every
// gradient buffer it writes (`bufs`); a null `used` means recompute.  forward: it needs `out`, and when it writes gradients
// (`grads`) every gradient buffer, the expected upstream gradients and the record to write.
static inline bool upstream_args_ok(int verify, const float* out, bool grads, bool bufs, const float* expected,
                                    const float* used) {
    return verify ? bufs : (out && (!grads || (bufs && expected && used)));
}

// ---------------------------------------------------------------------------------------------------------------
// Launch geometry of the persistent kernels, cached per (kernel, device).  The dynamic shared-memory opt-in belongs
// to the kernel in the current device's context, so a process that runs an operator on one device and then on
// another has to opt the kernel in on each.
// ---------------------------------------------------------------------------------------------------------------
constexpr int MAX_DEVICES = 64;  // device ordinals the caches can hold; a larger ordinal is B200RL_ERR_ARG

static inline int current_device(int& dev) {
    if (int rc = cuda_rc(cudaGetDevice(&dev))) return rc;
    return (dev >= 0 && dev < MAX_DEVICES) ? B200RL_OK : B200RL_ERR_ARG;
}

// let kernel K use `smem` bytes of dynamic shared memory on the current device (more than 48 KB needs the opt-in)
template <auto K>
static inline int smem_opt_in(size_t smem) {
    static size_t opted[MAX_DEVICES];  // largest size opted in so far
    if (smem <= 48 * 1024) return B200RL_OK;
    int dev = 0;
    if (int rc = current_device(dev)) return rc;
    if (smem <= opted[dev]) return B200RL_OK;
    if (int rc = cuda_rc(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem))) return rc;
    opted[dev] = smem;
    return B200RL_OK;
}

// SM count of the current device and CTAs of kernel K (threads, smem) resident per SM; opts K into `smem` first.
// B200RL_ERR_ARG if not even one CTA fits.  The occupancy is cached for the last smem size asked for on each device.
template <auto K>
static inline int resident_ctas(int threads, size_t smem, int& sm_count, int& per_sm) {
    static int sms[MAX_DEVICES];
    static size_t occ_smem[MAX_DEVICES];
    static int occ[MAX_DEVICES];  // 0 = not queried yet
    if (int rc = smem_opt_in<K>(smem)) return rc;
    int dev = 0;
    if (int rc = current_device(dev)) return rc;
    if (sms[dev] == 0)
        if (int rc = cuda_rc(cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev))) return rc;
    if (occ[dev] == 0 || occ_smem[dev] != smem) {
        if (int rc = cuda_rc(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[dev], K, threads, smem))) return rc;
        occ_smem[dev] = smem;
    }
    sm_count = sms[dev];
    per_sm = occ[dev];
    return per_sm < 1 ? B200RL_ERR_ARG : B200RL_OK;
}

// The instantiation table of the row-width-specialised kernels: f(std::integral_constant<int, N>{}) for
// N in {2..10, 12, 14, 16, 18}, f(std::integral_constant<int, 0>{}) (the generic kernel) for every other N.
template <class F>
static inline int with_nc(int n, F&& f) {
    switch (n) {
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 5: return f(std::integral_constant<int, 5>{});
        case 6: return f(std::integral_constant<int, 6>{});
        case 7: return f(std::integral_constant<int, 7>{});
        case 8: return f(std::integral_constant<int, 8>{});
        case 9: return f(std::integral_constant<int, 9>{});
        case 10: return f(std::integral_constant<int, 10>{});
        case 12: return f(std::integral_constant<int, 12>{});
        case 14: return f(std::integral_constant<int, 14>{});
        case 16: return f(std::integral_constant<int, 16>{});
        case 18: return f(std::integral_constant<int, 18>{});
        default: return f(std::integral_constant<int, 0>{});
    }
}

// per-CTA partial sums live in workspace words [WS_CTRL_WORDS, WS_PARTIAL_LIMIT_WORDS): above them sit the packed accumulators of
// grid_sum_fx and the scheduling counters of fused.cu, which must stay zero between launches
static inline bool ws_partials_fit(long long n_words, size_t ws_bytes) {
    return ws_bytes >= (size_t)WS_MIN_BYTES && (long long)WS_CTRL_WORDS + n_words <= (long long)WS_PARTIAL_LIMIT_WORDS;
}

// Loss reduction of the per-sample heads (the one-thread-per-row TD kernels and C51 of td.cu, FQF's fraction loss of
// quantile.cu): fin(k, total) receives the grid total of acc[k].  The one-round-trip grid_sum_fx when no last CTA is needed
// and the grid has at most FX_MAX_GRID CTAs; otherwise the ticket grid_sum, and the return value says whether this is the
// last CTA, which then sees every row's stores.  The host launches the NT > 128 builds only on such grids and never with
// need_last, so they compile only grid_sum_fx.
template <int K, int NT, class Fin>
__device__ __forceinline__ bool td_loss_sum(float (&acc)[K], float* ws, bool need_last, Fin fin) {
    if (NT > 128 || (!need_last && gridDim.x <= FX_MAX_GRID)) {
        grid_sum_fx<K, NT>(acc, ws, fin);
        return false;
    }
    double tot[K];
    const bool last = grid_sum<K, NT>(acc, tot, ws, 0);
    if (last && threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) fin(k, tot[k]);
    }
    return last;
}

// Launch plan of the per-sample heads (qntd, dqfd, soft_td, fqf_fraction); kern(std::integral_constant<int, NT>()) names
// the NT-thread build, and CTA x owns rows [x * NT, x * NT + NT).  Up to 1024 rows without a sequence priority -- the usual
// replay-buffer batch -- run as ONE CTA of 256 / 512 / 1024 threads, which reduces the loss without any grid round trip;
// anything else runs as 128-thread CTAs, whose K partial sums each must fit the workspace.
template <int K, class Args, class Kern>
static int launch_td_rows(Kern kern, const Args& a, long long rows, bool priority, float* ws, size_t ws_bytes,
                          cudaStream_t st) {
    const bool one_cta = rows <= 1024 && !priority;
    const long long grid = (rows + 127) / 128;
    if (!ws_partials_fit(one_cta ? 0 : grid * K, ws_bytes)) return B200RL_ERR_WORKSPACE;
    if (!one_cta) return launch_k(kern(std::integral_constant<int, 128>()), (int)grid, 128, 0, st, a, ws);
    if (rows <= 256) return launch_k(kern(std::integral_constant<int, 256>()), 1, 256, 0, st, a, ws);
    if (rows <= 512) return launch_k(kern(std::integral_constant<int, 512>()), 1, 512, 0, st, a, ws);
    return launch_k(kern(std::integral_constant<int, 1024>()), 1, 1024, 0, st, a, ws);
}

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace b200rl
