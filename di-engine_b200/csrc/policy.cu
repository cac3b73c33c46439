// The batch-level pieces that sit directly either side of the operators in the reference's policies (SURVEY section 8f rank 1):
//
//   PPOPolicy._forward_learn, ding/policy/ppo.py:274-306
//       value *= std; next_value *= std                                  (value_norm, :276-278; std = RunningMeanStd.std, a float)
//       adv = gae(gae_data(value, next_value, reward, done, traj_flag))  (:280-282 -- ONE sequence of n_sample steps, 1-D)
//       unnormalized_returns = value + adv                               (:284)
//       value = value / std; return = unnormalized_returns / std         (:286-288)
//       running_mean_std.update(unnormalized_returns.cpu().numpy())      (:289 -- host sync + full D2H copy in the reference)
//       adv = (adv - adv.mean()) / (adv.std() + 1e-8)   per train batch  (:304-306)
//
// Kernels
//   gae_seq_kernel        the 1-D call of the real PPO learner: ONE CTA; delta / f in the reference's operation order, then the
//                         sequence is cut at every traj_flag == 1 (f == 0 there, so the recurrence restarts: segments are
//                         independent) and every segment is scanned by its own lane -- bit-identical to the sequential loop,
//                         #segments-fold parallel (n_sample = 3200 = 8 envs x 400 steps -> >= 8 lanes x <= 400 steps instead of
//                         one lane x 3200); returns / value-norm / the RunningMeanStd batch statistics fused into the write-out.
//   returns_kernel        the same epilogue for (T, B) batches behind gae_ws_kernel: one elementwise pass + statistics.
//   adv_stats_kernel      {mean, std(unbiased) + 1e-8} of a batch in one launch; the PPO kernels apply the normalisation on load
//                         (ppo_math.cuh adv_in), normalize_kernel materialises it for callers that want the tensor.
#include <math.h>

#include "../../include/b200rl.h"
#include "policy_stats.cuh"

namespace b200rl {

// ---------------------------------------------------------------------------------------------------------------
// 1-D GAE with segment-parallel scan (single CTA, T <= GS_MAX_T)
// ---------------------------------------------------------------------------------------------------------------
constexpr int GS_NT = 1024;
constexpr int GS_MAX_T = 24576;  // 2 arrays x 4 B x T of dynamic shared memory (192 KB)

__global__ void __launch_bounds__(GS_NT) gae_seq_kernel(const float* __restrict__ value, float* __restrict__ next_value,
                                                       const float* __restrict__ reward, const float* __restrict__ done,
                                                       const float* __restrict__ traj, float* __restrict__ adv, int T,
                                                       float gamma, float gl, int mask_inplace, RetArgs ra) {
    pdl_prologue();
    extern __shared__ float s_seq[];
    float* s_d = s_seq;       // delta, then adv
    float* s_f = s_seq + T;   // trace factor
    __shared__ int s_nseg;
    __shared__ int s_cnt[GS_NT / 32];
    const int tid = threadIdx.x;
    const float vs = ra.vscale;
    // ---- phase 1: delta_t, f_t in the reference's operation order (gae.py:61-63), value_norm scaling first (ppo.py:276-278)
    for (int t = tid; t < T; t += GS_NT) {
        float v = value[t], nv = next_value[t];
        if (vs != 0.f) {
            v = fmul(v, vs);
            nv = fmul(nv, vs);
        }
        const float d = done ? done[t] : 0.f;
        const float tf = traj ? traj[t] : d;
        if (done) {
            nv = fmul(nv, fsub(1.f, d));
            if (mask_inplace && d != 0.f) next_value[t] = nv;
        }
        s_d[t] = fsub(fadd(reward[t], fmul(gamma, nv)), v);
        s_f[t] = fmul(gl, fsub(1.f, tf));
    }
    __syncthreads();
    // ---- phase 2: segment ends = positions whose factor is exactly 0 (the recurrence restarts there) and the last step,
    // compacted in order: count per contiguous strip of time steps, prefix over the CTA, write
    const int strip = (T + GS_NT - 1) / GS_NT;
    const int t0 = tid * strip, t1 = min(T, t0 + strip);
    int mine = 0;
    for (int t = t0; t < t1; ++t) mine += (s_f[t] == 0.f || t == T - 1) ? 1 : 0;
    // inclusive scan of `mine` over the CTA
    int incl = mine;
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) s_cnt[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int w = s_cnt[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += n;
        }
        s_cnt[lane] = w;
        if (lane == 31) s_nseg = w;
    }
    __syncthreads();
    const int base = incl - mine + (wid ? s_cnt[wid - 1] : 0);
    __shared__ int s_end[GS_NT];
    const int nseg = s_nseg;
    const bool fits = nseg <= GS_NT;
    if (fits) {
        int k = base;
        for (int t = t0; t < t1; ++t)
            if (s_f[t] == 0.f || t == T - 1) s_end[k++] = t;
    }
    __syncthreads();
    // ---- phase 3: lane s scans segment (end_{s-1}, end_s] backwards; separate mul / add: bit-identical to the torch loop
    if (fits) {
        if (tid < nseg) {
            const int hi = s_end[tid];
            const int lo = tid ? s_end[tid - 1] + 1 : 0;
            float carry = 0.f;  // the step after a segment end contributes f * carry with f == 0 -> +0 exactly as in the loop
            // 16 steps at a time: the shared-memory operands are in registers before the dependent chain needs them (a
            // load / compute / store loop would pay shared-memory latency on every step, far more than the chain's two
            // dependent floating-point operations)
            int t = hi;
            for (; t - 15 >= lo; t -= 16) {
                float d[16], f[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    d[k] = s_d[t - k];
                    f[k] = s_f[t - k];
                }
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    carry = fadd(d[k], fmul(f[k], carry));
                    d[k] = carry;
                }
#pragma unroll
                for (int k = 0; k < 16; ++k) s_d[t - k] = d[k];
            }
            for (; t >= lo; --t) {
                carry = fadd(s_d[t], fmul(s_f[t], carry));
                s_d[t] = carry;
            }
        }
    } else if (tid == 0) {  // more segments than lanes (T > 1024 with almost every step an episode end): sequential
        float carry = 0.f;
        for (int t = T - 1; t >= 0; --t) {
            carry = fadd(s_d[t], fmul(s_f[t], carry));
            s_d[t] = carry;
        }
    }
    __syncthreads();
    // ---- phase 4: write-out (+ returns, value-norm, statistics)
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int t = tid; t < T; t += GS_NT) {
        const float a = s_d[t];
        adv[t] = a;
        acc[2] += (double)a;
        acc[3] += (double)a * (double)a;
        if (ra.ret_unnorm || ra.value_out || ra.ret_out || ra.stats) {
            float v = value[t];
            if (vs != 0.f) v = fmul(v, vs);
            const float r = fadd(v, a);  // unnormalized_returns = value + adv (ppo.py:284)
            if (ra.ret_unnorm) ra.ret_unnorm[t] = r;
            if (ra.value_out) ra.value_out[t] = vs != 0.f ? __fdiv_rn(v, vs) : v;
            if (ra.ret_out) ra.ret_out[t] = vs != 0.f ? __fdiv_rn(r, vs) : r;
            acc[0] += (double)r;
            acc[1] += (double)r * (double)r;
        }
    }
    if (ra.stats || ra.adv_stats) {
        double tot[4];
        block_sum_d<4, GS_NT>(acc, tot);
        if (tid == 0) {
            const double n = (double)T, m = tot[0] / n;
            if (ra.stats) {
                ra.stats[0] = (float)m;
                ra.stats[1] = (float)fmax(tot[1] / n - m * m, 0.0);  // np.var: population variance
                ra.stats[2] = (float)n;
            }
            if (ra.adv_stats) write_adv_stats(ra.adv_stats, tot[2], tot[3], n);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// (T, B) epilogue behind gae_ws_kernel: returns / value-norm / statistics in one elementwise pass.
// The four sums (r, r^2, adv, adv^2) are reduced per CTA in fp64 and joined across CTAs with fp64 atomics; the CTA that
// arrives last writes the statistics (ret_stats_join).
// ---------------------------------------------------------------------------------------------------------------
template <bool VEC>
__global__ void __launch_bounds__(256) returns_kernel(const float* __restrict__ value, const float* __restrict__ adv,
                                                      long long n, RetArgs ra, double* __restrict__ ws_d,
                                                      unsigned int* __restrict__ ws_join) {
    pdl_prologue();
    const float vs = ra.vscale;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    if (VEC) {  // n % 4 == 0, 16-byte aligned tensors
        const long long n4 = n >> 2;
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
            const float4 v = reinterpret_cast<const float4*>(value)[i], a = reinterpret_cast<const float4*>(adv)[i];
            float4 ru, vo, ro;
            ret_one(vs, v.x, a.x, ru.x, vo.x, ro.x, acc);
            ret_one(vs, v.y, a.y, ru.y, vo.y, ro.y, acc);
            ret_one(vs, v.z, a.z, ru.z, vo.z, ro.z, acc);
            ret_one(vs, v.w, a.w, ru.w, vo.w, ro.w, acc);
            if (ra.ret_unnorm) reinterpret_cast<float4*>(ra.ret_unnorm)[i] = ru;
            if (ra.value_out) reinterpret_cast<float4*>(ra.value_out)[i] = vo;
            if (ra.ret_out) reinterpret_cast<float4*>(ra.ret_out)[i] = ro;
        }
    } else {
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
            float ru, vo, ro;
            ret_one(vs, value[i], adv[i], ru, vo, ro, acc);
            if (ra.ret_unnorm) ra.ret_unnorm[i] = ru;
            if (ra.value_out) ra.value_out[i] = vo;
            if (ra.ret_out) ra.ret_out[i] = ro;
        }
    }
    if (!ra.stats && !ra.adv_stats) return;
    ret_stats_join<256>(acc, ra, (double)n, ws_d, ws_join);
}

// ---------------------------------------------------------------------------------------------------------------
// advantage statistics {mean, std (unbiased, torch.std) + 1e-8} and the normalisation itself
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) adv_stats_kernel(const float* __restrict__ x, long long n, float* __restrict__ out,
                                                        double* __restrict__ ws_d, unsigned int* __restrict__ ws_join) {
    pdl_prologue();
    double acc[2] = {0.0, 0.0};
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const double v = (double)x[i];
        acc[0] += v;
        acc[1] += v * v;
    }
    double tot[2];
    block_sum_d<2, 256>(acc, tot);
    if (threadIdx.x != 0) return;
    double s1 = tot[0], s2 = tot[1];
    if (gridDim.x > 1) {
        atomicAdd(ws_d, s1);
        atomicAdd(ws_d + 1, s2);
        __threadfence();
        if (atomicAdd(ws_join, 1u) != gridDim.x - 1) return;
        __threadfence();
        s1 = atomicAdd(ws_d, 0.0);
        s2 = atomicAdd(ws_d + 1, 0.0);
        ws_d[0] = 0.0;
        ws_d[1] = 0.0;
        *ws_join = 0u;
    }
    write_adv_stats(out, s1, s2, (double)n);
}

__global__ void __launch_bounds__(256) normalize_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                                        long long n, float* __restrict__ out) {
    pdl_prologue();
    const float m = stats[0], d = stats[1];
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        out[i] = __fdiv_rn(fsub(x[i], m), d);
}

// ---------------------------------------------------------------------------------------------------------------
// IMPALAPolicy._reshape_data masking (ding/policy/impala.py:316-322), one elementwise launch:
//   weights_ = 1 - done;  values[1:] *= weights_;  weights = ones; weights[1:] = weights_[:-1];  rewards *= weights
// backward: d/d values[t] = g[t] * (1 - done[t-1]) for t >= 1 (the in-place product of the reference), same kernel shape.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) impala_mask_kernel(const float* __restrict__ values, const float* __restrict__ rewards,
                                                          const float* __restrict__ done, long long T, long long B,
                                                          float* __restrict__ values_out, float* __restrict__ rewards_out,
                                                          float* __restrict__ weights_out) {
    pdl_prologue();
    const long long n = (T + 1) * B;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const long long t = i / B;
        const float m = t >= 1 ? fsub(1.f, done[i - B]) : 1.f;  // 1 - done[t-1]
        values_out[i] = t >= 1 ? fmul(values[i], m) : values[i];
        if (t < T) {
            if (weights_out) weights_out[i] = m;
            if (rewards_out) rewards_out[i] = fmul(rewards[i], m);
        }
    }
}

}  // namespace b200rl

using namespace b200rl;

namespace b200rl {
int gae_scan(const float* value, float* next_value, const float* reward, const float* done, const float* traj_flag, float* adv,
             long long T, long long C, long long A, double gamma_d, double lambda_d, int mask_next_value_inplace,
             float vscale, void* stream);
}

// workspace words used by the two-sum joins above: 4 doubles + 2 counters right after the packed accumulators of grid_sum_fx
static double* ws_doubles(float* ws) { return reinterpret_cast<double*>(ws + WS_FX_OFF_WORDS + 32); }
static unsigned int* ws_joins(float* ws) { return reinterpret_cast<unsigned int*>(ws + WS_FX_OFF_WORDS + 48); }

extern "C" int b200rl_adv_stats(const float* x, long long n, float* stats2, float* workspace, size_t workspace_bytes,
                                void* stream) {
    if (!x || !stats2 || !workspace || n < 1 || workspace_bytes < WS_MIN_BYTES) return B200RL_ERR_ARG;
    long long grid = div_up(n, 256 * 8);
    if (grid > NUM_SMS * 4) grid = NUM_SMS * 4;
    if (grid < 1) grid = 1;
    return launch_k(adv_stats_kernel, (int)grid, 256, 0, (cudaStream_t)stream, x, n, stats2, ws_doubles(workspace),
                    ws_joins(workspace));
}

extern "C" int b200rl_normalize(const float* x, const float* stats2, long long n, float* out, void* stream) {
    if (!x || !stats2 || !out || n < 0) return B200RL_ERR_ARG;
    if (n == 0) return B200RL_OK;
    long long grid = div_up(n, 256 * 4);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    return launch_k(normalize_kernel, (int)grid, 256, 0, (cudaStream_t)stream, x, stats2, n, out);
}

extern "C" int b200rl_gae_returns(const float* value, float* next_value, const float* reward, const float* done,
                                  const float* traj_flag, long long T, long long C, long long A, double gamma,
                                  double lambda_, int mask_next_value_inplace, double value_scale, float* adv,
                                  float* unnormalized_return, float* value_out, float* return_out, float* stats3,
                                  float* adv_stats2, float* workspace, size_t workspace_bytes, void* stream) {
    if (T < 1 || C < 1 || A < 1 || !value || !next_value || !reward || !adv || !workspace ||
        workspace_bytes < WS_MIN_BYTES || value_scale < 0.0)
        return B200RL_ERR_ARG;
    RetArgs ra{};
    ra.vscale = (float)value_scale;
    ra.ret_unnorm = unnormalized_return; ra.value_out = value_out; ra.ret_out = return_out; ra.stats = stats3;
    ra.adv_stats = adv_stats2;
    cudaStream_t st = (cudaStream_t)stream;
    if (C == 1 && T <= GS_MAX_T) {  // the real PPO learner's call: one sequence, everything in one launch
        const size_t smem = (size_t)2 * T * sizeof(float);
        if (int rc = smem_opt_in<gae_seq_kernel>(smem)) return rc;
        return launch_k(gae_seq_kernel, 1, GS_NT, smem, st, value, next_value, reward, done, traj_flag, adv, (int)T,
                        (float)gamma, (float)(gamma * lambda_), mask_next_value_inplace, ra);
    }
    // (T, B): the streaming scan (value_norm scaling applied on load), then one elementwise epilogue launch (returns_kernel).
    const bool want_epi = unnormalized_return || value_out || return_out || stats3 || adv_stats2;
    int rc = gae_scan(value, next_value, reward, done, traj_flag, adv, T, C, A, gamma, lambda_, mask_next_value_inplace,
                      (float)value_scale, stream);
    if (rc != 0 || !want_epi) return rc;
    const long long n = T * C;
    const bool vec = (n % 4 == 0) && aligned16(value) && aligned16(adv) && (!unnormalized_return || aligned16(unnormalized_return)) &&
                     (!value_out || aligned16(value_out)) && (!return_out || aligned16(return_out));
    long long grid = div_up(n, 256 * (vec ? 8 : 4));
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    if (vec)
        return launch_k(returns_kernel<true>, (int)grid, 256, 0, st, value, (const float*)adv, n, ra, ws_doubles(workspace),
                        ws_joins(workspace));
    return launch_k(returns_kernel<false>, (int)grid, 256, 0, st, value, (const float*)adv, n, ra, ws_doubles(workspace),
                    ws_joins(workspace));
}

/* rewards / rewards_out / weights_out nullable (the backward pass masks a gradient with values = g, the other outputs off) */
extern "C" int b200rl_impala_mask(const float* values, const float* rewards, const float* done, long long T, long long B,
                                  float* values_out, float* rewards_out, float* weights_out, void* stream) {
    if (!values || !done || !values_out || T < 1 || B < 1 || (rewards_out && !rewards)) return B200RL_ERR_ARG;
    long long grid = div_up((T + 1) * B, 256 * 4);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    return launch_k(impala_mask_kernel, (int)grid, 256, 0, (cudaStream_t)stream, values, rewards, done, T, B, values_out,
                    rewards_out, weights_out);
}
