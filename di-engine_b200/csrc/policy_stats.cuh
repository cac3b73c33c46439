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
};

// {mean, torch.std (unbiased) + 1e-8} from the fp64 sums of x and x^2
__device__ __forceinline__ void write_adv_stats(float* out, double s1, double s2, double nn) {
    const double m = s1 / nn;
    const double var = (s2 - s1 * m) / (nn - 1.0);  // n == 1 -> nan, as torch.std
    const double sd = var != var ? var : sqrt(fmax(var, 0.0));
    out[0] = (float)m;
    out[1] = fadd((float)sd, 1e-8f);
}


// the element-wise part of the epilogue for one (value, adv) pair: unnormalized return, stored value / return, the four sums
__device__ __forceinline__ void ret_one(float vs, float v, float a, float& ru, float& vo, float& ro, double (&acc)[4]) {
    if (vs != 0.f) v = fmul(v, vs);
    const float r = fadd(v, a);  // unnormalized_returns = value + adv (ppo.py:284)
    ru = r;
    vo = vs != 0.f ? __fdiv_rn(v, vs) : v;
    ro = vs != 0.f ? __fdiv_rn(r, vs) : r;
    acc[0] += (double)r;
    acc[1] += (double)r * (double)r;
    acc[2] += (double)a;
    acc[3] += (double)a * (double)a;
}

// CTA partial sums -> workspace doubles (fp64 atomics: order-dependent in the last bits of a double only; the results are rounded
// to fp32), the CTA that arrives last writes the statistics and re-zeroes the workspace words
template <int NT>
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
        ra.stats[1] = (float)fmax(s[1] / nn - m * m, 0.0);  // np.var: population variance
        ra.stats[2] = (float)nn;
    }
    if (ra.adv_stats) write_adv_stats(ra.adv_stats, s[2], s[3], nn);
    *ws_join = 0u;
}

}  // namespace b200rl
