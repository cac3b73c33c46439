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
// (unnormalized_returns = value + adv, ppo.py:284 / ppof.py:195), stored value / return, and the sums of the return the
// statistics describe (PPOPolicy: the unnormalised one; PPOF: the stored one)
template <int VN>
__device__ __forceinline__ void ret_encode(float vs, float v, float a, float& ru, float& vo, float& ro, double (&acc)[4]) {
    const float r = fadd(v, a);
    ru = r;
    vo = vn_encode<VN>(v, vs);
    ro = vn_encode<VN>(r, vs);
    const float s = VN == VN_PPO ? r : ro;
    acc[0] += (double)s;
    acc[1] += (double)s * (double)s;
}

// {mean, torch.std (unbiased) + 1e-8} from the fp64 sums of x and x^2
__device__ __forceinline__ void write_adv_stats(float* out, double s1, double s2, double nn) {
    const double m = s1 / nn;
    const double var = (s2 - s1 * m) / (nn - 1.0);  // n == 1 -> nan, as torch.std
    const double sd = var != var ? var : sqrt(fmax(var, 0.0));
    out[0] = (float)m;
    out[1] = fadd((float)sd, 1e-8f);
}


// the element-wise part of the (T, B) epilogue for one (value, adv) pair: the value as returns_kernel reads it (raw for the
// scaling modes, already decoded by the decode pass for the others), then ret_encode, then the advantage sums
template <int VN>
__device__ __forceinline__ void ret_one(float vs, float v, float a, float& ru, float& vo, float& ro, double (&acc)[4]) {
    if constexpr (VN == VN_PPO || VN == VN_BASELINE) v = vn_decode<VN>(v, vs);
    ret_encode<VN>(vs, v, a, ru, vo, ro, acc);
    acc[2] += (double)a;
    acc[3] += (double)a * (double)a;
}

// np.var (population variance) from the fp64 sums: the PPO build clamps a NaN to 0, as it always has; PPOF's modes keep it,
// as np.var of returns holding a NaN or an inf gives NaN
template <int VN>
__device__ __forceinline__ double pop_var(double v) {
    return (VN != VN_PPO && v != v) ? v : fmax(v, 0.0);
}

// CTA partial sums -> workspace doubles (fp64 atomics: order-dependent in the last bits of a double only; the results are rounded
// to fp32), the CTA that arrives last writes the statistics and re-zeroes the workspace words
template <int NT, int VN>
__device__ __forceinline__ void ret_stats_join(double (&acc)[4], const RetArgs& ra, double nn, double* ws_d,
                                               unsigned int* ws_join) {
    double tot[4];
    block_sum_d<4, NT>(acc, tot);
    if (threadIdx.x != 0) return;
#pragma unroll
    for (int k = 0; k < 4; ++k) atomicAdd(ws_d + k, tot[k]);
    __threadfence();
    if (atomicAdd(ws_join, 1u) != gridDim.x - 1) return;
    __threadfence();
    double s[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        s[k] = atomicAdd(ws_d + k, 0.0);
        ws_d[k] = 0.0;
    }
    const double m = s[0] / nn;
    if (ra.stats) {
        ra.stats[0] = (float)m;
        ra.stats[1] = (float)pop_var<VN>(s[1] / nn - m * m);
        ra.stats[2] = (float)nn;
    }
    if (ra.adv_stats) write_adv_stats(ra.adv_stats, s[2], s[3], nn);
    *ws_join = 0u;
}

}  // namespace b200rl
