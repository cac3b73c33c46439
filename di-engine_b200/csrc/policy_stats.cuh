#pragma once
// Used by policy.cu: the batch-level pieces PPOPolicy wraps around gae (ding/policy/ppo.py:274-306) -- returns,
// value-norm scaling and the two sets of batch statistics -- as an epilogue argument block plus its reductions.
#include <math.h>

#include "common.cuh"

namespace b200rl {

template <class T>
__device__ __forceinline__ T warp_sum_t(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// CTA-wide sum of K doubles per thread; result valid in thread 0 (fixed order: deterministic)
template <int K, int NT>
__device__ __forceinline__ void block_sum_d(double (&v)[K], double (&tot)[K]) {
    __shared__ double s_bs[K][NT / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const double r = warp_sum_t(v[k]);
        if (lane == 0) s_bs[k][wid] = r;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double r = 0.0;
            for (int w = 0; w < NT / 32; ++w) r += s_bs[k][w];
            tot[k] = r;
        }
    }
    __syncthreads();
}

struct RetArgs {
    float vscale;      // 0: no value_norm
    float* ret_unnorm;  // nullable
    float* value_out;   // nullable: (value*s)/s
    float* ret_out;     // nullable: unnormalized / s
    float* stats;       // nullable: {mean, population variance, count} of the unnormalized returns (RunningMeanStd.update input)
    float* adv_stats;   // nullable: {mean, std(unbiased) + 1e-8} of adv (ppo.py:304-306 when the whole batch is one minibatch)
    const float* mu;     // VN_POPART: the PopArt head's mu / sigma, one device float each
    const float* sigma;
};

// ---------------------------------------------------------------------------------------------------------------
// Value normalisation around gae.  VN_PPO is PPOPolicy's (value scaled by ra.vscale when it is not 0, statistics of the
// unnormalised return).  The other four are PPOFPolicy's value_norm modes (ding/policy/ppof.py:171-208), in the order of
// the C ABI's value_norm argument:
//   VN_BASELINE  value * std on load, / std on store; statistics of the STORED return (ppof.py:206-208 divides in place)
//   VN_RESCALE   h^-1 on load, h on store (value_rescale.py:4-34, eps = 1e-2)
//   VN_SYMLOG    inv_symlog on load, symlog on store (value_rescale.py:37-66)
//   VN_POPART    reward -> (reward - mu) / sigma on load, value as it is (ppof.py:171-179)
// Every expression is the reference's torch expression, one rounded fp32 operation per torch op, in its order.
// ---------------------------------------------------------------------------------------------------------------
enum ValueNorm : int { VN_BASELINE = 0, VN_RESCALE = 1, VN_SYMLOG = 2, VN_POPART = 3, VN_PPO = 4 };

// torch.sign: (0 < x) - (x < 0), so sign(NaN) = sign(-0) = 0
__device__ __forceinline__ float vn_sign(float x) { return (float)((0.f < x) - (x < 0.f)); }

// value_transform: sign(x) * (sqrt(|x| + 1) - 1) + eps * x
__device__ __forceinline__ float vn_h(float x) {
    return fadd(fmul(vn_sign(x), fsub(__fsqrt_rn(fadd(fabsf(x), 1.f)), 1.f)), fmul(0.01f, x));
}
// value_inv_transform: sign(x) * (((sqrt(1 + 4 eps ((|x| + 1) + eps)) - 1) / (2 eps)) ** 2 - 1); 4 eps and 2 eps are python
// doubles rounded to fp32 scalars, and the division by a python scalar is a true division
__device__ __forceinline__ float vn_h_inv(float x) {
    const float u = __fdiv_rn(fsub(__fsqrt_rn(fadd(1.f, fmul(0.04f, fadd(fadd(fabsf(x), 1.f), 0.01f)))), 1.f), 0.02f);
    return fmul(vn_sign(x), fsub(fmul(u, u), 1.f));
}
// symlog: sign(x) * log(|x| + 1)  (logf of |x| + 1, as torch.log computes it, not log1pf)
__device__ __forceinline__ float vn_symlog(float x) { return fmul(vn_sign(x), logf(fadd(fabsf(x), 1.f))); }
// inv_symlog: sign(x) * (exp(|x|) - 1)
__device__ __forceinline__ float vn_inv_symlog(float x) { return fmul(vn_sign(x), fsub(expf(fabsf(x)), 1.f)); }

// the critic's output as gae sees it, for a kernel that reads the raw value (VN_POPART decodes the reward instead)
template <int VN>
__device__ __forceinline__ float vn_decode(float v, float vs) {
    if constexpr (VN == VN_PPO || VN == VN_BASELINE) return vs != 0.f ? fmul(v, vs) : v;
    else if constexpr (VN == VN_RESCALE) return vn_h_inv(v);
    else if constexpr (VN == VN_SYMLOG) return vn_inv_symlog(v);
    else return v;
}

// the stored form of a decoded value or return
template <int VN>
__device__ __forceinline__ float vn_encode(float v, float vs) {
    if constexpr (VN == VN_PPO || VN == VN_BASELINE) return vs != 0.f ? __fdiv_rn(v, vs) : v;
    else if constexpr (VN == VN_RESCALE) return vn_h(v);
    else if constexpr (VN == VN_SYMLOG) return vn_symlog(v);
    else return v;
}

// the element-wise part of the epilogue for a DECODED value v and its advantage a: unnormalized return
// (unnormalized_returns = value + adv, ppo.py:284 / ppof.py:195) and stored value / return; returns the value the return
// statistics describe (PPOPolicy: the unnormalised return; PPOF: the stored one)
template <int VN>
__device__ __forceinline__ float ret_encode(float vs, float v, float a, float& ru, float& vo, float& ro) {
    const float r = fadd(v, a);
    ru = r;
    vo = vn_encode<VN>(v, vs);
    ro = vn_encode<VN>(r, vs);
    return VN == VN_PPO ? r : ro;
}

// ---------------------------------------------------------------------------------------------------------------
// Batch statistics.  Every kernel accumulates, per statistic, the fp64 sums of (x - p) and (x - p)^2 around a pivot p: one
// element of the batch (element 0, 0 when it is not finite), the same in every thread.  The plain sums of x and x^2 lose
// (mean / sd)^2 of the double's precision to cancellation in S2/n - m^2 -- all of fp32's with a mean 1e4 sd away.  With a
// pivot from the batch, (p - mean)^2 <= n * var, so the loss is bounded by the batch size, whatever the offset.
// Per-CTA sums are joined across the grid in a fixed order (stats_grid_join): bit-identical from run to run.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double stats_pivot(float x0) { return isfinite(x0) ? (double)x0 : 0.0; }

// A global load that stays behind pdl_prologue's griddepcontrol.wait.  The compiler may hoist a loop-invariant load through
// a const __restrict__ pointer above it (it takes the data as read-only for the kernel's lifetime): with plain value[0] /
// adv[0] loads, the sm_90a build of returns_kernel issued both as LDG.E.CONSTANT ahead of PREEXIT / ACQBULK, so the pivot was
// read before gae_scan -- which writes adv[0] last -- had finished, and the statistics changed from run to run.  __ldcg is
// not such a load; the compiler keeps it behind the wait.
__device__ __forceinline__ float ld_after_wait(const float* p) { return __ldcg(p); }

__device__ __forceinline__ void moments_add(double& s1, double& s2, float x, double p) {
    const double d = (double)x - p;
    s1 += d;
    s2 = fma(d, d, s2);
}

// the decoded value of a value returns_kernel reads: raw for the scaling modes, already decoded by the decode pass for the
// others
template <int VN>
__device__ __forceinline__ float ret_value(float v, float vs) {
    if constexpr (VN == VN_PPO || VN == VN_BASELINE) return vn_decode<VN>(v, vs);
    else return v;
}

// (T, B) epilogue element: ret_encode of the decoded value, then the shifted sums of the return (acc[0..1], pivot pv[0]) and
// of adv (acc[2..3], pv[1])
template <int VN>
__device__ __forceinline__ void ret_one(float vs, float v, float a, float& ru, float& vo, float& ro, double (&acc)[4],
                                        const double (&pv)[2]) {
    moments_add(acc[0], acc[1], ret_encode<VN>(vs, ret_value<VN>(v, vs), a, ru, vo, ro), pv[0]);
    moments_add(acc[2], acc[3], a, pv[1]);
}

// the pivots of the shifted sums: element 0's statistics source and advantage, from its DECODED value v0 (the value
// ret_encode receives for element 0: the pivot must be a member of the batch)
template <int VN>
__device__ __forceinline__ void ret_pivots(float vs, float v0, float a0, double (&pv)[2]) {
    float ru, vo, ro;
    pv[0] = stats_pivot(ret_encode<VN>(vs, v0, a0, ru, vo, ro));
    pv[1] = stats_pivot(a0);
}

// Grid-wide totals of K per-thread fp64 sums.  Thread 0 of every CTA stores the CTA's sums to the workspace's partial rows
// (part[blockIdx.x * K + k]) and takes a ticket; the CTA that draws the last one adds the rows in a fixed order (thread i:
// rows i, i + NT, ...; then block_sum_d) and resets the ticket.  Returns true in thread 0 of that CTA, which then holds the
// totals in tot.  A one-CTA grid touches neither the rows nor the ticket.
template <int K, int NT>
__device__ __forceinline__ bool stats_grid_join(double (&acc)[K], double (&tot)[K], double* part, unsigned int* ticket) {
    __shared__ bool s_last;
    block_sum_d<K, NT>(acc, tot);
    if (gridDim.x == 1) return threadIdx.x == 0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) part[(size_t)blockIdx.x * K + k] = tot[k];
        __threadfence();
        s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return false;
    __threadfence();
    double v[K];
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = 0.0;
    for (unsigned int b = threadIdx.x; b < gridDim.x; b += NT)
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] += __ldcg(part + (size_t)b * K + k);
    block_sum_d<K, NT>(v, tot);
    if (threadIdx.x == 0) *ticket = 0u;
    return threadIdx.x == 0;
}

// {mean, torch.std (unbiased) + 1e-8} from the shifted sums s1 = sum(x - p), s2 = sum((x - p)^2)
__device__ __forceinline__ void write_adv_stats(float* out, double s1, double s2, double p, double nn) {
    const double d = s1 / nn;
    const double var = (s2 - s1 * d) / (nn - 1.0);  // n == 1 -> nan, as torch.std
    const double sd = var != var ? var : sqrt(fmax(var, 0.0));
    out[0] = (float)(p + d);
    out[1] = fadd((float)sd, 1e-8f);
}

// np.var (population variance) from the shifted sums: the PPO build clamps a NaN to 0, as it always has; PPOF's modes keep
// it, as np.var of returns holding a NaN or an inf gives NaN
template <int VN>
__device__ __forceinline__ double pop_var(double v) {
    return (VN != VN_PPO && v != v) ? v : fmax(v, 0.0);
}

// the statistics of gae_seq_kernel / returns_kernel from the grid totals of ret_one's four sums
template <int VN>
__device__ __forceinline__ void write_ret_stats(const RetArgs& ra, const double (&tot)[4], const double (&pv)[2],
                                                double nn) {
    if (ra.stats) {
        const double d = tot[0] / nn;
        ra.stats[0] = (float)(pv[0] + d);
        ra.stats[1] = (float)pop_var<VN>(tot[1] / nn - d * d);
        ra.stats[2] = (float)nn;
    }
    if (ra.adv_stats) write_adv_stats(ra.adv_stats, tot[2], tot[3], pv[1], nn);
}

}  // namespace b200rl
