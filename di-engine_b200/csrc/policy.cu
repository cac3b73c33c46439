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
// gae_seq_kernel and returns_kernel are templated on the value normalisation (policy_stats.cuh): VN_PPO is the above, the
// other four are PPOFPolicy's value_norm modes (ding/policy/ppof.py:160-210, b200rl_gae_returns_norm).  value_map_kernel is
// symlog / inv_symlog and the decode pass of PPOF's (T, B) path; value_map_bwd_kernel the autograd of the first two.
#include <math.h>

#include "../../include/b200rl.h"
#include "policy_stats.cuh"

namespace b200rl {

// ---------------------------------------------------------------------------------------------------------------
// 1-D GAE with segment-parallel scan (single CTA, T <= GS_MAX_T)
// ---------------------------------------------------------------------------------------------------------------
constexpr int GS_NT = 1024;
constexpr int GS_MAX_T = 24576;  // 2 arrays x 4 B x T of dynamic shared memory (192 KB)

// VN: the value normalisation around gae (policy_stats.cuh), decoded in phase 1 and encoded in phase 4
template <int VN>
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
    float mu = 0.f, sigma = 1.f;
    if constexpr (VN == VN_POPART) {
        mu = *ra.mu;
        sigma = *ra.sigma;
    }
    // ---- phase 1: delta_t, f_t in the reference's operation order (gae.py:61-63), value_norm decoding first (ppo.py:276-278,
    // ppof.py:171-189)
    for (int t = tid; t < T; t += GS_NT) {
        const float v = vn_decode<VN>(value[t], vs);
        float nv = vn_decode<VN>(next_value[t], vs);
        float r = reward[t];
        if constexpr (VN == VN_POPART) r = __fdiv_rn(fsub(r, mu), sigma);
        const float d = done ? done[t] : 0.f;
        const float tf = traj ? traj[t] : d;
        if (done) {
            nv = fmul(nv, fsub(1.f, d));
            if (VN == VN_PPO && mask_inplace && d != 0.f) next_value[t] = nv;
        }
        s_d[t] = fsub(fadd(r, fmul(gamma, nv)), v);
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
    if constexpr (VN != VN_PPO) {
        // The loop carries 0 * adv[t + 1] across a segment end t, so a non-finite adv[t + 1] there makes adv[0 .. t] NaN; the
        // lanes above restarted from 0.  Take the last such end and poison everything up to it, as the loop does.  (The PPO
        // build keeps the lane result there, the deviation DESIGN.md documents for gae.)
        __shared__ int s_cut;
        if (tid == 0) s_cut = -1;
        __syncthreads();
        int cut = -1;
        for (int t = tid; t < T - 1; t += GS_NT)
            if (s_f[t] == 0.f && !isfinite(s_d[t + 1])) cut = t;
        if (cut >= 0) atomicMax(&s_cut, cut);
        __syncthreads();
        const int c = s_cut;
        for (int t = tid; t <= c; t += GS_NT) s_d[t] = __int_as_float(0x7fc00000);
        __syncthreads();
    }
    // ---- phase 4: write-out (+ returns, value-norm, statistics around element 0's pivots)
    double acc[4] = {0.0, 0.0, 0.0, 0.0}, pv[2];
    ret_pivots<VN>(vs, vn_decode<VN>(ld_after_wait(value), vs), s_d[0], pv);
    for (int t = tid; t < T; t += GS_NT) {
        const float a = s_d[t];
        adv[t] = a;
        moments_add(acc[2], acc[3], a, pv[1]);
        if (ra.ret_unnorm || ra.value_out || ra.ret_out || ra.stats) {
            float ru, vo, ro;
            moments_add(acc[0], acc[1], ret_encode<VN>(vs, vn_decode<VN>(value[t], vs), a, ru, vo, ro), pv[0]);
            if (ra.ret_unnorm) ra.ret_unnorm[t] = ru;
            if (ra.value_out) ra.value_out[t] = vo;
            if (ra.ret_out) ra.ret_out[t] = ro;
        }
    }
    if (ra.stats || ra.adv_stats) {
        double tot[4];
        if (stats_grid_join<4, GS_NT>(acc, tot, nullptr, nullptr)) write_ret_stats<VN>(ra, tot, pv, (double)T);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// (T, B) epilogue behind gae_ws_kernel: returns / value-norm / statistics in one elementwise pass.  The scaling modes read the
// raw value; the others read the value the decode pass (value_map_kernel) wrote.
// The four shifted sums of r and adv (ret_one) are reduced per CTA in fp64 and joined across CTAs in a fixed order; the CTA
// that arrives last writes the statistics (stats_grid_join, write_ret_stats).
// ---------------------------------------------------------------------------------------------------------------
template <int VN, bool VEC>
__global__ void __launch_bounds__(256) returns_kernel(const float* __restrict__ value, const float* __restrict__ adv,
                                                      long long n, RetArgs ra, double* __restrict__ ws_part,
                                                      unsigned int* __restrict__ ws_join) {
    pdl_prologue();
    const float vs = ra.vscale;
    double acc[4] = {0.0, 0.0, 0.0, 0.0}, pv[2];
    // the first element of each thread is loaded together with the pivots, so that their latency is paid once
    const long long stride = (long long)gridDim.x * 256;
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (VEC) {  // n % 4 == 0, 16-byte aligned tensors
        const long long n4 = n >> 2;
        const float4* v4 = reinterpret_cast<const float4*>(value);
        const float4* a4 = reinterpret_cast<const float4*>(adv);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f), a = v;
        if (i < n4) {
            v = v4[i];
            a = a4[i];
        }
        ret_pivots<VN>(vs, ret_value<VN>(ld_after_wait(value), vs), ld_after_wait(adv), pv);
        for (; i < n4; i += stride) {
            float4 ru, vo, ro;
            ret_one<VN>(vs, v.x, a.x, ru.x, vo.x, ro.x, acc, pv);
            ret_one<VN>(vs, v.y, a.y, ru.y, vo.y, ro.y, acc, pv);
            ret_one<VN>(vs, v.z, a.z, ru.z, vo.z, ro.z, acc, pv);
            ret_one<VN>(vs, v.w, a.w, ru.w, vo.w, ro.w, acc, pv);
            if (ra.ret_unnorm) reinterpret_cast<float4*>(ra.ret_unnorm)[i] = ru;
            if (ra.value_out) reinterpret_cast<float4*>(ra.value_out)[i] = vo;
            if (ra.ret_out) reinterpret_cast<float4*>(ra.ret_out)[i] = ro;
            if (i + stride < n4) {
                v = v4[i + stride];
                a = a4[i + stride];
            }
        }
    } else {
        float v = 0.f, a = 0.f;
        if (i < n) {
            v = value[i];
            a = adv[i];
        }
        ret_pivots<VN>(vs, ret_value<VN>(ld_after_wait(value), vs), ld_after_wait(adv), pv);
        for (; i < n; i += stride) {
            float ru, vo, ro;
            ret_one<VN>(vs, v, a, ru, vo, ro, acc, pv);
            if (ra.ret_unnorm) ra.ret_unnorm[i] = ru;
            if (ra.value_out) ra.value_out[i] = vo;
            if (ra.ret_out) ra.ret_out[i] = ro;
            if (i + stride < n) {
                v = value[i + stride];
                a = adv[i + stride];
            }
        }
    }
    if (!ra.stats && !ra.adv_stats) return;
    double tot[4];
    if (stats_grid_join<4, 256>(acc, tot, ws_part, ws_join)) write_ret_stats<VN>(ra, tot, pv, (double)n);
}

// ---------------------------------------------------------------------------------------------------------------
// advantage statistics {mean, std (unbiased, torch.std) + 1e-8} and the normalisation itself
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) adv_stats_kernel(const float* __restrict__ x, long long n, float* __restrict__ out,
                                                        double* __restrict__ ws_part, unsigned int* __restrict__ ws_join) {
    pdl_prologue();
    const double p = stats_pivot(ld_after_wait(x));
    double acc[2] = {0.0, 0.0};
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        moments_add(acc[0], acc[1], x[i], p);
    double tot[2];
    if (stats_grid_join<2, 256>(acc, tot, ws_part, ws_join)) write_adv_stats(out, tot[0], tot[1], p, (double)n);
}

__global__ void __launch_bounds__(256) normalize_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                                        long long n, float* __restrict__ out) {
    pdl_prologue();
    const float m = ld_after_wait(stats), d = ld_after_wait(stats + 1);  // adv_stats_kernel wrote them just before
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

// ---------------------------------------------------------------------------------------------------------------
// Element-wise value maps: symlog / inv_symlog forward and backward (value_rescale.py:37-66), and the decode pass of a
// PPOF advantage recompute that does not fit gae_seq_kernel -- h^-1 or inv_symlog of value and next_value (two arrays in one
// launch), or PopArt's (reward - mu) / sigma (ppof.py:177).
// ---------------------------------------------------------------------------------------------------------------
enum ValueMap : int { VM_SYMLOG = 0, VM_INV_SYMLOG = 1, VM_H_INV = 2, VM_POPART_REWARD = 3 };

template <int M>
__device__ __forceinline__ float value_map(float x, float mu, float sigma) {
    if constexpr (M == VM_SYMLOG) return vn_symlog(x);
    else if constexpr (M == VM_INV_SYMLOG) return vn_inv_symlog(x);
    else if constexpr (M == VM_H_INV) return vn_h_inv(x);
    else return __fdiv_rn(fsub(x, mu), sigma);
}

// y0 = map(x0) and, when x1 is given, y1 = map(x1); mu / sigma: device floats, read only by VM_POPART_REWARD
template <int M>
__global__ void __launch_bounds__(256) value_map_kernel(const float* __restrict__ x0, float* __restrict__ y0,
                                                        const float* __restrict__ x1, float* __restrict__ y1, long long n,
                                                        const float* __restrict__ mu, const float* __restrict__ sigma) {
    pdl_prologue();
    float m = 0.f, sg = 1.f;
    if constexpr (M == VM_POPART_REWARD) {
        m = *mu;
        sg = *sigma;
    }
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        y0[i] = value_map<M>(x0[i], m, sg);
        if (x1) y1[i] = value_map<M>(x1[i], m, sg);
    }
}

// torch autograd of the reference expressions, op by op (sign contributes a zero gradient, accumulated last):
//   symlog      sign(x) * log(|x| + 1):  dx = 0 + ((g * sign(x)) / (|x| + 1)) * sign(x)
//   inv_symlog  sign(x) * (exp(|x|) - 1): dx = 0 + ((g * sign(x)) * exp(|x|)) * sign(x)
template <int M>
__global__ void __launch_bounds__(256) value_map_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                            float* __restrict__ dx, long long n) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const float xi = x[i], s = vn_sign(xi), gs = fmul(g[i], s);
        const float d = M == VM_SYMLOG ? __fdiv_rn(gs, fadd(fabsf(xi), 1.f)) : fmul(gs, expf(fabsf(xi)));
        dx[i] = fadd(0.f, fmul(d, s));
    }
}

}  // namespace b200rl

using namespace b200rl;

namespace b200rl {
int gae_scan(const float* value, float* next_value, const float* reward, const float* done, const float* traj_flag, float* adv,
             long long T, long long C, long long A, double gamma_d, double lambda_d, int mask_next_value_inplace,
             float vscale, void* stream);
}

// workspace of the statistics joins above: the per-CTA rows of fp64 sums (at most NUM_SMS * 8 CTAs x 4 doubles) in the partial
// region, and the ticket right after the packed accumulators of grid_sum_fx
static double* ws_stats_part(float* ws) { return reinterpret_cast<double*>(ws + WS_CTRL_WORDS); }
static unsigned int* ws_joins(float* ws) { return reinterpret_cast<unsigned int*>(ws + WS_FX_OFF_WORDS + 48); }
static_assert(WS_CTRL_WORDS % 2 == 0 && WS_CTRL_WORDS + NUM_SMS * 8 * 4 * 2 <= WS_PARTIAL_LIMIT_WORDS,
              "the statistics rows fit the workspace's partial region");

extern "C" int b200rl_adv_stats(const float* x, long long n, float* stats2, float* workspace, size_t workspace_bytes,
                                void* stream) {
    if (!x || !stats2 || !workspace || n < 1 || workspace_bytes < WS_MIN_BYTES) return B200RL_ERR_ARG;
    long long grid = div_up(n, 256 * 8);
    if (grid > NUM_SMS * 4) grid = NUM_SMS * 4;
    if (grid < 1) grid = 1;
    return launch_k(adv_stats_kernel, (int)grid, 256, 0, (cudaStream_t)stream, x, n, stats2, ws_stats_part(workspace),
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
        if (int rc = smem_opt_in<gae_seq_kernel<VN_PPO>>(smem)) return rc;
        return launch_k(gae_seq_kernel<VN_PPO>, 1, GS_NT, smem, st, value, next_value, reward, done, traj_flag, adv, (int)T,
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
        return launch_k(returns_kernel<VN_PPO, true>, (int)grid, 256, 0, st, value, (const float*)adv, n, ra,
                        ws_stats_part(workspace), ws_joins(workspace));
    return launch_k(returns_kernel<VN_PPO, false>, (int)grid, 256, 0, st, value, (const float*)adv, n, ra,
                    ws_stats_part(workspace), ws_joins(workspace));
}

// ---- PPOFPolicy's advantage recompute (ding/policy/ppof.py:160-210) -----------------------------------------------------------
static long long map_grid(long long n) {
    long long grid = div_up(n, 256 * 4);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    return grid < 1 ? 1 : grid;
}

template <int VN>
static int launch_gae_seq(const float* value, const float* next_value, const float* reward, const float* done,
                          const float* traj_flag, float* adv, long long T, double gamma, double lambda_, const RetArgs& ra,
                          cudaStream_t st) {
    const size_t smem = (size_t)2 * T * sizeof(float);
    if (int rc = smem_opt_in<gae_seq_kernel<VN>>(smem)) return rc;
    return launch_k(gae_seq_kernel<VN>, 1, GS_NT, smem, st, value, const_cast<float*>(next_value), reward, done, traj_flag,
                    adv, (int)T, (float)gamma, (float)(gamma * lambda_), 0, ra);
}

template <int VN>
static int launch_returns(const float* value, const float* adv, long long n, const RetArgs& ra, float* workspace,
                          cudaStream_t st) {
    const bool vec = (n % 4 == 0) && aligned16(value) && aligned16(adv) && (!ra.value_out || aligned16(ra.value_out)) &&
                     (!ra.ret_out || aligned16(ra.ret_out));
    long long grid = div_up(n, 256 * (vec ? 8 : 4));
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    if (vec)
        return launch_k(returns_kernel<VN, true>, (int)grid, 256, 0, st, value, adv, n, ra, ws_stats_part(workspace),
                        ws_joins(workspace));
    return launch_k(returns_kernel<VN, false>, (int)grid, 256, 0, st, value, adv, n, ra, ws_stats_part(workspace),
                    ws_joins(workspace));
}

// (T, C) or a sequence longer than GS_MAX_T: decode pass (not for baseline: gae_scan scales on load), gae_scan, the mode's
// returns_kernel
template <int VN>
static int launch_gae_returns_tc(const float* value, const float* next_value, const float* reward, const float* done,
                                 const float* traj_flag, float* adv, long long T, long long C, double gamma, double lambda_,
                                 const RetArgs& ra, float* scratch, float* workspace, cudaStream_t st) {
    const long long n = T * C;
    const float* v = value;
    const float* nv = next_value;
    const float* r = reward;
    int rc = 0;
    if constexpr (VN == VN_RESCALE || VN == VN_SYMLOG) {
        constexpr int M = VN == VN_RESCALE ? VM_H_INV : VM_INV_SYMLOG;
        rc = launch_k(value_map_kernel<M>, (int)map_grid(n), 256, 0, st, value, scratch, next_value, scratch + n, n,
                      (const float*)nullptr, (const float*)nullptr);
        v = scratch;
        nv = scratch + n;
    } else if constexpr (VN == VN_POPART) {
        rc = launch_k(value_map_kernel<VM_POPART_REWARD>, (int)map_grid(n), 256, 0, st, reward, scratch,
                      (const float*)nullptr, (float*)nullptr, n, ra.mu, ra.sigma);
        r = scratch;
    }
    if (rc) return rc;
    // mask_next_value_inplace = 0: next_value is only read
    rc = gae_scan(v, const_cast<float*>(nv), r, done, traj_flag, adv, T, C, 1, gamma, lambda_, 0,
                  VN == VN_BASELINE ? ra.vscale : 0.f, st);
    if (rc || !(ra.value_out || ra.ret_out || ra.stats || ra.adv_stats)) return rc;
    return launch_returns<VN>(v, adv, n, ra, workspace, st);
}

template <int VN>
static int gae_returns_norm(const float* value, const float* next_value, const float* reward, const float* done,
                            const float* traj_flag, float* adv, long long T, long long C, double gamma, double lambda_,
                            const RetArgs& ra, float* scratch, float* workspace, cudaStream_t st) {
    if (C == 1 && T <= GS_MAX_T)  // every PPOF call: one sequence of n_sample steps, one launch
        return launch_gae_seq<VN>(value, next_value, reward, done, traj_flag, adv, T, gamma, lambda_, ra, st);
    return launch_gae_returns_tc<VN>(value, next_value, reward, done, traj_flag, adv, T, C, gamma, lambda_, ra, scratch,
                                     workspace, st);
}

extern "C" int b200rl_gae_returns_norm(const float* value, const float* next_value, const float* reward, const float* done,
                                       const float* traj_flag, long long T, long long C, double gamma, double lambda_,
                                       int value_norm, double std, const float* popart_mu, const float* popart_sigma,
                                       float* adv, float* value_out, float* return_out, float* stats3, float* adv_stats2,
                                       float* scratch, float* workspace, size_t workspace_bytes, void* stream) {
    if (T < 1 || C < 1 || !value || !next_value || !reward || !adv || !workspace || workspace_bytes < WS_MIN_BYTES)
        return B200RL_ERR_ARG;
    if (value_norm < VN_BASELINE || value_norm > VN_POPART) return B200RL_ERR_ARG;
    if (value_norm == VN_BASELINE && !(std > 0.0)) return B200RL_ERR_ARG;
    if (value_norm == VN_POPART && (!popart_mu || !popart_sigma)) return B200RL_ERR_ARG;
    const bool one_launch = C == 1 && T <= GS_MAX_T;
    if (!one_launch && value_norm != VN_BASELINE && !scratch) return B200RL_ERR_ARG;
    RetArgs ra{};
    ra.vscale = value_norm == VN_BASELINE ? (float)std : 0.f;
    ra.value_out = value_out; ra.ret_out = return_out; ra.stats = stats3; ra.adv_stats = adv_stats2;
    ra.mu = popart_mu; ra.sigma = popart_sigma;
    cudaStream_t st = (cudaStream_t)stream;
    switch (value_norm) {
        case VN_BASELINE:
            return gae_returns_norm<VN_BASELINE>(value, next_value, reward, done, traj_flag, adv, T, C, gamma, lambda_, ra,
                                                 scratch, workspace, st);
        case VN_RESCALE:
            return gae_returns_norm<VN_RESCALE>(value, next_value, reward, done, traj_flag, adv, T, C, gamma, lambda_, ra,
                                                scratch, workspace, st);
        case VN_SYMLOG:
            return gae_returns_norm<VN_SYMLOG>(value, next_value, reward, done, traj_flag, adv, T, C, gamma, lambda_, ra,
                                               scratch, workspace, st);
        default:
            return gae_returns_norm<VN_POPART>(value, next_value, reward, done, traj_flag, adv, T, C, gamma, lambda_, ra,
                                               scratch, workspace, st);
    }
}

extern "C" int b200rl_value_map_fwd(int mode, const float* x, long long n, float* y, void* stream) {
    if (n < 0 || (mode != VM_SYMLOG && mode != VM_INV_SYMLOG)) return B200RL_ERR_ARG;
    if (n == 0) return B200RL_OK;
    if (!x || !y) return B200RL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = (int)map_grid(n);
    if (mode == VM_SYMLOG)
        return launch_k(value_map_kernel<VM_SYMLOG>, grid, 256, 0, st, x, y, (const float*)nullptr, (float*)nullptr, n,
                        (const float*)nullptr, (const float*)nullptr);
    return launch_k(value_map_kernel<VM_INV_SYMLOG>, grid, 256, 0, st, x, y, (const float*)nullptr, (float*)nullptr, n,
                    (const float*)nullptr, (const float*)nullptr);
}

extern "C" int b200rl_value_map_bwd(int mode, const float* x, const float* g, long long n, float* dx, void* stream) {
    if (n < 0 || (mode != VM_SYMLOG && mode != VM_INV_SYMLOG)) return B200RL_ERR_ARG;
    if (n == 0) return B200RL_OK;
    if (!x || !g || !dx) return B200RL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = (int)map_grid(n);
    if (mode == VM_SYMLOG) return launch_k(value_map_bwd_kernel<VM_SYMLOG>, grid, 256, 0, st, x, g, dx, n);
    return launch_k(value_map_bwd_kernel<VM_INV_SYMLOG>, grid, 256, 0, st, x, g, dx, n);
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
