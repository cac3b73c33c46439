// n-step TD heads of ding/rl_utils/td.py:
//   q_nstep_td_error (:649-719) / q_nstep_td_error_with_rescale (:810-867), bdq_nstep_td_error and
//   R2D2's sequence loss (ding/policy/r2d2.py)                               -> qntd_fwd / qntd_bwd
//   dqfd_nstep_td_error (:870-983, with rescale :986-1090) and R2D3's sequence loop -> dqfd_fwd / dqfd_bwd
//   m_q_1step_td_error, q_nstep_sql_td_error, q_v_1step_td_error             -> soft_td_fwd / qntd_bwd
//   dist_nstep_td_error (C51 projection, :413-523)                           -> dntd_fwd / dntd_bwd
//   generalized_lambda_returns / multistep_forward_view (:1574-1651), td_lambda_error (:1539-1571) and the
//   UPGO return (upgo.py:46-68)                                              -> lambda_returns (+ fused TD(lambda) head)
// Each reference call is ~20-35 tiny torch launches plus an autograd backward; here it is one forward and one
// backward launch.  These batches are small (B ~ 32..512): latency, not bandwidth, is what the kernels minimise.
// qntd, dqfd and soft_td run one thread per row and share the n-step return and the one-hot gradient store below, and the
// loss reduction and host launch plan of common.cuh (td_loss_sum, launch_td_rows); only their targets differ.
#include <math.h>

#include <type_traits>

#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {

// ---------------------------------------------------------------------------------------------------------------
// value rescaling h / h^-1 (value_rescale.py:4-34), evaluated in the reference's operation order
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sgn(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }
__device__ __forceinline__ float value_h(float x, float eps) {
    return fadd(fmul(sgn(x), fsub(__fsqrt_rn(fadd(fabsf(x), 1.f)), 1.f)), fmul(eps, x));
}
__device__ __forceinline__ float value_h_inv(float x, float eps, float four_eps, float two_eps) {
    float t = fadd(fadd(fabsf(x), 1.f), eps);
    float u = __fdiv_rn(fsub(__fsqrt_rn(fadd(1.f, fmul(four_eps, t))), 1.f), two_eps);
    return fmul(sgn(x), fsub(fmul(u, u), 1.f));
}

// elementwise criteria (reduction='none'): value and d/d(input)
__device__ __forceinline__ float criterion_eval(int kind, float param, float x, float y, float& dx) {
    const float d = x - y, ad = fabsf(d);
    switch (kind) {
        case 0: dx = 2.f * d; return d * d;                                        // nn.MSELoss
        case 1: dx = sgn(d); return ad;                                            // nn.L1Loss
        case 2:                                                                    // nn.SmoothL1Loss(beta)
            if (ad < param) { dx = d / param; return 0.5f * d * d / param; }
            dx = sgn(d); return ad - 0.5f * param;
        default:                                                                   // nn.HuberLoss(delta)
            if (ad <= param) { dx = d; return 0.5f * d * d; }
            dx = param * sgn(d); return param * (ad - 0.5f * param);
    }
}

// The first min(n, 8) rewards of one sample, rw[i * Bi], into registers.  Callers issue this together with their other
// per-sample loads, before any of them is used: a load inside the n-step loop is one L2 round trip per step.
__device__ __forceinline__ void nstep_reward_load(float (&rwv)[8], const float* __restrict__ rw, size_t Bi, int n) {
#pragma unroll
    for (int i = 0; i < 8; ++i) rwv[i] = i < n ? rw[i * Bi] : 0.f;
}

// sum_i reward[i] * gamma^i over the nstep rewards of one sample (td.py:261-265 / :277-281, matmul(reward_factor, reward)
// :453-456): the first 8 come from nstep_reward_load, the rest are read at rw[i * Bi]; rf returns gamma^nstep as the loop
// builds it (reward_factor[nstep]).
__device__ __forceinline__ float nstep_reward_sum(const float (&rwv)[8], const float* __restrict__ rw, size_t Bi, int nstep,
                                                  float g, float& rf) {
    float ret = 0.f;
    rf = 1.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (i < nstep) {
            ret = fadd(ret, fmul(rwv[i], rf));
            rf = fmul(g, rf);
        }
    }
    for (int i = 8; i < nstep; ++i) {
        ret = fadd(ret, fmul(rw[i * Bi], rf));
        rf = fmul(g, rf);
    }
    return ret;
}

// The CTA's gradient rows [r0, r0 + NT) of g (R rows of N): row r0 + t, staged by thread t, is coef0[t] at idx0[t] (plus
// coef1[t] at idx1[t] when given) and zero elsewhere.  The rows are contiguous, so the CTA stores them together, coalesced.
template <int NT>
__device__ __forceinline__ void store_onehot_rows(float* __restrict__ g, long long r0, long long R, int N, const float* coef0,
                                                  const int* idx0, const float* coef1 = nullptr, const int* idx1 = nullptr) {
    __syncthreads();
    const long long rows = (R - r0) < NT ? (R - r0) : NT;
    float* gq = g + r0 * N;
    for (long long i = threadIdx.x; i < rows * N; i += NT) {
        const int rr = (int)(i / N), j = (int)(i - (long long)rr * N);
        float v = (j == idx0[rr]) ? coef0[rr] : 0.f;
        if (coef1) v += (j == idx1[rr]) ? coef1[rr] : 0.f;
        gq[i] = v;
    }
}

// The scalars that qntd, dqfd and soft_td derive alike on the host (td_scalars below).
struct TdScalars {
    float gamma, gamma_pow_n;
    float eps, four_eps, two_eps;  // value rescaling (qntd, dqfd)
    double loss_div;               // loss = sum(w*td) / loss_div
    // sequence form (qntd, dqfd): priority[b] = max_w*max_t e + mean_w*sum_t e / prio_div over the per-step errors e
    float prio_max_w, prio_mean_w, prio_div;
};

struct QntdArgs : TdScalars {
    const float* q;            // (S, G, N)
    const float* next_q;       // (S, G, N)
    const long long* action;   // (S, G)
    const long long* next_action;
    const float* reward;       // (nstep, S), (S) when cum_reward; sequence form (S = Tseq*Bcol): (Tseq, nstep, Bcol)
    const float* done;         // (S)
    const float* weight;       // (S) or null
    const float* value_gamma;  // null, or pointer with stride 0 (0-dim) / 1 (S)
    long long value_gamma_stride;
    const float* gamma_ps;     // NGU per-sample gamma (Bcol) or null
    long long S;               // samples
    long long Bcol;            // == S, or the batch width of the sequence form (sample s = t*Bcol + b)
    int G;                     // rows per sample: 1, the agent dim of the multi-agent form or the BDQ branches
    int N;
    int nstep;
    int cum_reward;
    int rescale;
    int criterion;
    float crit_param;
    int group_mean;    // td_error_per_sample (S) = mean over the G rows (bdq_nstep_td_error, td.py:788) instead of (S, G)
    float* loss;
    float* td_err;
    float* dcrit;      // (S, G) d criterion / d q_sa (unweighted): what the backward launch needs
    float* target;     // nullable: the (detached) n-step target (S, G), for callers that apply their own criterion
    float* grad_unit;  // nullable (S, G, N): d loss / d q for a unit upstream gradient, written by the forward launch
    float* priority;   // nullable (Bcol): sequence form only
};

// One launch: n-step target, criterion, deterministic loss reduction, per-sample errors AND (grad_unit) the gradient of the
// loss for a unit upstream gradient -- the backward launch only has to verify that the upstream gradient was 1.
template <int NT>
__global__ void __launch_bounds__(NT) qntd_fwd_kernel(QntdArgs a, float* ws) {
    pdl_prologue();
    __shared__ float s_coef[NT];
    __shared__ int s_act[NT];
    const long long s0 = (long long)blockIdx.x * NT;
    const long long s = s0 + threadIdx.x;
    const float inv_div = (float)(1.0 / a.loss_div);
    float acc[1] = {0.f};
    s_coef[threadIdx.x] = 0.f;
    s_act[threadIdx.x] = -1;
    if (s < a.S) {
        const long long tq_ = s / a.Bcol, b = s - tq_ * a.Bcol;  // sequence step / batch column (tq_ = 0 when Bcol == S)
        // every per-sample operand is requested before any is used, the action indices first: q[action] waits on them
        const int act0 = (int)a.action[s * a.G], nact0 = (int)a.next_action[s * a.G];
        const float* __restrict__ rw = a.cum_reward ? a.reward + s : a.reward + tq_ * a.nstep * a.Bcol + b;
        const size_t Bi = (size_t)a.Bcol;
        float rwv[8];
        nstep_reward_load(rwv, rw, Bi, a.cum_reward ? 1 : a.nstep);
        const float dn = a.done[s];
        const float w = a.weight ? a.weight[s] : 1.f;
        const float vgl = a.value_gamma ? a.value_gamma[s * a.value_gamma_stride] : a.gamma_pow_n;
        const float g = a.gamma_ps ? a.gamma_ps[b] : a.gamma;
        const float q0 = a.q[s * a.G * a.N + act0], nq0 = a.next_q[s * a.G * a.N + nact0];
        const float nd = fsub(1.f, dn);
        float ret = 0.f, vg;
        if (a.cum_reward) {
            ret = rwv[0];
            vg = vgl;
        } else {
            float rf;
            ret = nstep_reward_sum(rwv, rw, Bi, a.nstep, g, rf);
            vg = a.gamma_ps ? rf : vgl;  // reward_factor[nstep] for the NGU list-gamma form
        }
        float td_sum = 0.f;
        for (int gi = 0; gi < a.G; ++gi) {
            const long long r = s * a.G + gi;
            const int act = gi == 0 ? act0 : (int)a.action[r];
            const float q_sa = gi == 0 ? q0 : a.q[r * a.N + act];
            float tq = gi == 0 ? nq0 : a.next_q[r * a.N + a.next_action[r]];
            if (a.rescale) tq = value_h_inv(tq, a.eps, a.four_eps, a.two_eps);
            float target = fadd(ret, fmul(fmul(vg, tq), nd));  // td.py:266 / :273 / :282 / :712-715
            if (a.rescale) target = value_h(target, a.eps);
            float dx;
            const float td = criterion_eval(a.criterion, a.crit_param, q_sa, target, dx);
            if (a.group_mean) td_sum += td;
            else a.td_err[r] = td;
            if (a.target) a.target[r] = target;
            a.dcrit[r] = dx;
            acc[0] += td * w;
            if (a.grad_unit) {
                const float coef = w * dx * inv_div;
                if (a.G == 1) {
                    s_coef[threadIdx.x] = coef;
                    s_act[threadIdx.x] = act;
                } else {
                    float* gq = a.grad_unit + r * a.N;
                    for (int j = 0; j < a.N; ++j) gq[j] = (j == act) ? coef : 0.f;
                }
            }
        }
        if (a.group_mean) a.td_err[s] = td_sum / (float)a.G;
    }
    if (a.grad_unit && a.G == 1) store_onehot_rows<NT>(a.grad_unit, s0, a.S, a.N, s_coef, s_act);
    const bool last = td_loss_sum<1, NT>(acc, ws, a.priority, [&](int, double t) { a.loss[0] = (float)(t / a.loss_div); });
    if (last && a.priority) {
        // sequence form (ding/policy/r2d2.py:367-369): the last CTA sees every per-step error (published before the tickets)
        const long long Tq = a.S / a.Bcol;
        for (long long b = threadIdx.x; b < a.Bcol; b += NT) {
            float mx = 0.f, sm = 0.f;
            for (long long t = 0; t < Tq; ++t) {
                const float e = fabsf(__ldcg(a.td_err + t * a.Bcol + b));
                mx = (t == 0) ? e : fmaxf(mx, e);
                sm += e;
            }
            a.priority[b] = a.prio_max_w * mx + a.prio_mean_w * (sm / a.prio_div);
        }
    }
}

// grad_q[r, j] = 1[j == a_r] * (g_loss * w_s / loss_div + g_td) * dcrit[r].  skip_if_unit: the forward launch already wrote
// grad_q for g_loss == 1 and no per-sample upstream gradient -- verify on the device and leave at once if that held.
__global__ void qntd_bwd_kernel(const float* __restrict__ dcrit, const float* __restrict__ weight,
                                const long long* __restrict__ action, const float* __restrict__ g_loss,
                                const float* __restrict__ g_td, long long S, int G, int N, int group_mean, float inv_div,
                                int skip_if_unit, float* __restrict__ grad_q) {
    pdl_prologue();
    const float g = g_loss ? *g_loss : 0.f;
    if (skip_if_unit && !g_td && g == 1.f) return;
    const long long n = S * G * N;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / N;
        const int j = (int)(i - r * N);
        float out = 0.f;
        if (j == (int)action[r]) {
            const long long s = r / G;
            float c = g * (weight ? weight[s] : 1.f) * inv_div;
            if (g_td) c += group_mean ? g_td[s] / (float)G : g_td[r];
            out = c * dcrit[r];
        }
        grad_q[i] = out;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// DQfD: n-step TD + 1-step TD + supervised large-margin loss (td.py:870-983, with rescale :986-1090), and R2D3's per-step
// loop over it (ding/policy/r2d3.py:322-388) as the sequence form.  Per sample:
//   td_n = crit(q_sa, nstep target), td_1 = crit(q_sa, 1-step target), JE = is_expert * (max_j(q_j + m*[j != a]) - q_sa)
//   loss = mean(w * (ln*td_n + l1*td_1 + ls*JE)),  per-sample = ln*|td_n| + l1*|td_1| + ls*|JE|,  stats = means of the three
// ---------------------------------------------------------------------------------------------------------------
struct DqfdArgs : TdScalars {
    const float* q;           // (S, N)
    const float* next_q;      // (S, N)
    const float* next_q1;     // (S, N) new_n_q_one_step
    const long long* action;  // (S)
    const long long* next_action;
    const long long* next_action1;
    const float* reward;      // (nstep, S), (S) when cum_reward; sequence form (S = Tseq*Bcol): (Tseq, nstep, Bcol)
    const float* done;        // (S)
    const float* done1;       // (S) done_one_step
    const float* weight;      // (S) or null
    const float* value_gamma; // null, or stride 0 (0-dim) / 1 (S); n-step target only (td.py:955)
    long long value_gamma_stride;
    const float* is_expert;   // (S)
    long long S;
    long long Bcol;           // == S, or the batch width of the sequence form (sample s = t*Bcol + b)
    int N;
    int nstep;
    int cum_reward;
    int rescale;
    int criterion;            // criterion_eval kind, or -1: no TD terms (the caller applies its own criterion to target_n/1)
    float crit_param;
    float lam_n, lam_1, lam_s, margin;
    float* loss;
    float* td_err;            // (S)
    float* stats;             // (3): td_n, td_1, JE, each sum / loss_div
    float4* saved;            // (S): d crit_n, d crit_1, is_expert, argmax | sign codes << 24 -- what the backward launch needs
    float* target_n;          // nullable (S): the detached targets, for callers that apply their own criterion
    float* target_1;
    float* grad_unit;         // nullable (S, N): d loss / d q for a unit upstream gradient
    float* priority;          // nullable (Bcol): sequence form only
};

__device__ __forceinline__ int sgn_code(float x) { return x > 0.f ? 2 : (x < 0.f ? 0 : 1); }  // sgn(x) + 1

template <int NT>
__global__ void __launch_bounds__(NT) dqfd_fwd_kernel(DqfdArgs a, float* ws) {
    pdl_prologue();
    __shared__ float s_ca[NT], s_ck[NT];  // unit-gradient coefficient at the action / at the margin argmax
    __shared__ int s_act[NT], s_k[NT];
    const long long s0 = (long long)blockIdx.x * NT;
    const long long s = s0 + threadIdx.x;
    const float inv_div = (float)(1.0 / a.loss_div);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    s_ca[threadIdx.x] = s_ck[threadIdx.x] = 0.f;
    s_act[threadIdx.x] = s_k[threadIdx.x] = -1;
    if (s < a.S) {
        const long long tq_ = s / a.Bcol, b = s - tq_ * a.Bcol;
        // every per-sample operand is requested before any is used, the action indices first: q[action] waits on them
        const int act = (int)a.action[s], nact = (int)a.next_action[s], nact1 = (int)a.next_action1[s];
        const float* __restrict__ rw = a.cum_reward ? a.reward + s : a.reward + tq_ * a.nstep * a.Bcol + b;
        const size_t Bi = (size_t)a.Bcol;
        float rwv[8];
        nstep_reward_load(rwv, rw, Bi, a.cum_reward ? 1 : a.nstep);
        // cum_reward: reward[0].unsqueeze(0) is sample 0's reward, broadcast to every sample (td.py:954, :958)
        const float r1c = a.cum_reward ? a.reward[0] : 0.f;
        const float dn = a.done[s], dn1 = a.done1[s];
        const float w = a.weight ? a.weight[s] : 1.f;
        const float vgl = a.value_gamma ? a.value_gamma[s * a.value_gamma_stride] : a.gamma_pow_n;
        const float ie = a.is_expert[s];
        const float* __restrict__ qr = a.q + s * a.N;
        const float q_sa = qr[act], nq = a.next_q[s * a.N + nact], nq1 = a.next_q1[s * a.N + nact1];
        // supervised margin term: max_j(q_j + l_j), l = margin except 0 at the action (td.py:969-972); the gradient of the max
        // goes to the FIRST maximal index, as torch.max(dim=1) returns it (a NaN is maximal: the first NaN)
        float mx = 0.f;
        int k = 0;
        for (int j0 = 0; j0 < a.N; j0 += 4) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = j0 + u < a.N ? qr[j0 + u] : 0.f;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int j = j0 + u;
                if (j < a.N) {
                    const float x = fadd(v[u], j == act ? 0.f : a.margin);
                    if (j == 0 || x > mx || (x != x && mx == mx)) {
                        mx = x;
                        k = j;
                    }
                }
            }
        }
        const float je = fmul(ie, fsub(mx, q_sa));
        // n-step target (td.py:943-949 / :1045-1054)
        float tq = nq, tq1 = nq1;
        if (a.rescale) {
            tq = value_h_inv(tq, a.eps, a.four_eps, a.two_eps);
            tq1 = value_h_inv(tq1, a.eps, a.four_eps, a.two_eps);
        }
        float ret;
        if (a.cum_reward) {
            ret = rwv[0];
        } else {
            float rf;
            ret = nstep_reward_sum(rwv, rw, Bi, a.nstep, a.gamma, rf);
        }
        float tn = fadd(ret, fmul(fmul(vgl, tq), fsub(1.f, dn)));
        // 1-step target: reward[0], gamma ** 1, never value_gamma (td.py:953-964 / :1058-1069)
        float t1 = fadd(a.cum_reward ? r1c : rwv[0], fmul(fmul(a.gamma, tq1), fsub(1.f, dn1)));
        if (a.rescale) {
            tn = value_h(tn, a.eps);
            t1 = value_h(t1, a.eps);
        }
        if (a.target_n) a.target_n[s] = tn;
        if (a.target_1) a.target_1[s] = t1;
        float dxn = 0.f, dx1 = 0.f, tdn = 0.f, td1 = 0.f;
        if (a.criterion >= 0) {
            tdn = criterion_eval(a.criterion, a.crit_param, q_sa, tn, dxn);
            td1 = criterion_eval(a.criterion, a.crit_param, q_sa, t1, dx1);
        }
        const float comb = fadd(fadd(fmul(a.lam_n, tdn), fmul(a.lam_1, td1)), fmul(a.lam_s, je));  // td.py:974-979
        a.td_err[s] = fadd(fadd(fmul(a.lam_n, fabsf(tdn)), fmul(a.lam_1, fabsf(td1))), fmul(a.lam_s, fabsf(je)));
        acc[0] = fmul(comb, w);
        acc[1] = tdn;
        acc[2] = td1;
        acc[3] = je;
        const int code = sgn_code(tdn) | (sgn_code(td1) << 2) | (sgn_code(je) << 4);
        a.saved[s] = make_float4(dxn, dx1, ie, __int_as_float(k | (code << 24)));
        if (a.grad_unit) {
            const float c = w * inv_div;
            s_ca[threadIdx.x] = c * (a.lam_n * dxn + a.lam_1 * dx1 - a.lam_s * ie);
            s_ck[threadIdx.x] = c * a.lam_s * ie;
            s_act[threadIdx.x] = act;
            s_k[threadIdx.x] = k;
        }
    }
    if (a.grad_unit) store_onehot_rows<NT>(a.grad_unit, s0, a.S, a.N, s_ca, s_act, s_ck, s_k);
    const bool last = td_loss_sum<4, NT>(acc, ws, a.priority, [&](int kk, double t) {
        const float v = (float)(t / a.loss_div);
        if (kk == 0) a.loss[0] = v;
        else a.stats[kk - 1] = v;
    });
    if (last && a.priority) {
        // sequence form (r2d3.py:386-388): the per-sample errors are already sums of absolute values, no abs here
        const long long Tq = a.S / a.Bcol;
        for (long long b = threadIdx.x; b < a.Bcol; b += NT) {
            float mx = 0.f, sm = 0.f;
            for (long long t = 0; t < Tq; ++t) {
                const float e = __ldcg(a.td_err + t * a.Bcol + b);
                mx = (t == 0) ? e : fmaxf(mx, e);
                sm = fadd(sm, e);
            }
            a.priority[b] = fadd(fmul(a.prio_max_w, mx), fmul(a.prio_mean_w, __fdiv_rn(sm, a.prio_div)));
        }
    }
}

// grad_q for arbitrary upstream gradients of the loss (g_loss), the per-sample error (g_td, (S)) and the three statistics
// (g_sn, g_s1, g_sje); each nullable = 0.  skip_if_unit: grad_q already holds the forward's unit-loss gradient -- verify on the
// device that only g_loss == 1 arrived and leave at once.
__global__ void dqfd_bwd_kernel(const float4* __restrict__ saved, const float* __restrict__ weight,
                                const long long* __restrict__ action, const float* __restrict__ g_loss,
                                const float* __restrict__ g_td, const float* __restrict__ g_sn, const float* __restrict__ g_s1,
                                const float* __restrict__ g_sje, long long S, int N, float lam_n, float lam_1, float lam_s,
                                float inv_div, int skip_if_unit, float* __restrict__ grad_q) {
    pdl_prologue();
    const float g = g_loss ? *g_loss : 0.f;
    if (skip_if_unit && !g_td && !g_sn && !g_s1 && !g_sje && g == 1.f) return;
    const float gn = g_sn ? *g_sn * inv_div : 0.f, g1 = g_s1 ? *g_s1 * inv_div : 0.f, gj = g_sje ? *g_sje * inv_div : 0.f;
    const long long n = S * N;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long s = i / N;
        const int j = (int)(i - s * N);
        const int act = (int)action[s];
        const float4 r = saved[s];
        const int bits = __float_as_int(r.w), k = bits & 0xffffff, code = bits >> 24;
        float out = 0.f;
        if (j == act || j == k) {
            const float sn = (float)((code & 3) - 1), s1 = (float)(((code >> 2) & 3) - 1), sj = (float)(((code >> 4) & 3) - 1);
            const float gt = g_td ? g_td[s] : 0.f;
            const float cl = g * (weight ? weight[s] : 1.f) * inv_div;
            // d / d q_sa of the TD terms, and d / d (max - q_sa) of the margin term, per unit of each output
            const float ctd = cl * (lam_n * r.x + lam_1 * r.y) + gt * (lam_n * sn * r.x + lam_1 * s1 * r.y) + gn * r.x + g1 * r.y;
            const float cje = (cl * lam_s + gt * lam_s * sj + gj) * r.z;
            if (j == act) out = ctd - cje;
            if (j == k) out += cje;
        }
        grad_q[i] = out;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The TD losses of the entropy-regularised value learners, one thread per row.  Only the target differs between modes:
//   MODE 0 Munchausen (m_q_1step_td_error, td.py:119-158):
//          r + alpha*clamp(log pi(a), -1, 1) + gamma * sum_j pi'_j * (q'_j - tau*log pi'_j) * (1 - d),
//          pi = softmax(target_q / tau), pi' = softmax(next_q / tau), each with its row max taken out first;
//   MODE 1 soft n-step (q_nstep_sql_td_error, :1219-1245): the n-step return of V' = alpha*logsumexp(next_n_q / alpha)
//          (+inf -> 20, -inf -> -20);
//   MODE 2 value 1-step (q_v_1step_td_error, :198-219): gamma*(1 - d)*v + r.
// Gathering q_sa, the criterion, the loss sum and the record qntd_bwd_kernel reads (dcrit, and the unit gradient) are those of
// qntd_fwd_kernel; every target is detached, so the gradient reaches q through q_sa alone.
// ---------------------------------------------------------------------------------------------------------------
struct SoftTdArgs : TdScalars {
    const float* q;           // (R, N)
    const float* target_q;    // MODE 0: (R, N), the target network on the current observation
    const float* next_q;      // MODE 0 / 1: (R, N); MODE 2: the state value v (R)
    const long long* action;  // (R)
    const float* reward;      // MODE 1: (nstep, S), (S) when cum_reward; MODE 0 / 2: (S)
    const float* done;        // (S)
    const float* weight;      // (R) or null
    const float* value_gamma; // MODE 1: null, or stride 0 (0-dim) / 1 (S)
    long long value_gamma_stride;
    long long R;              // rows
    int G;                    // rows per sample (S = R / G): reward and done of row r are sample r / G's
    int N;
    int nstep;
    float tau, alpha;
    int cum_reward;
    int criterion;
    float crit_param;
    float* loss;
    float* td_err;            // (R)
    float* dcrit;             // (R) d criterion / d q_sa: what qntd_bwd_kernel reads (G = 1 there)
    float* target;            // nullable (R): the detached target, for callers that apply their own criterion
    float* grad_unit;         // nullable (R, N): d loss / d q for a unit upstream gradient
    float* action_gap;        // MODE 0: sum(top1 - top2) / loss_div
    float* clipfrac;          // MODE 0 (R): 1 where log pi(a) was clamped
    float* record_v;          // MODE 1, nullable (R): V' before the return is formed
};

// torch.logsumexp over a row y(0..n) (ATen logsumexp_out_impl): m = amax(y), NaN propagating, taken as 0 when it is
// infinite; the result is log(sum_j exp(y_j - m)) + m.  m and the sum are returned too: softmax(y) = exp(y - m) / sum
// wherever m is finite.
template <class F>
__device__ __forceinline__ float row_logsumexp(F y, int n, float& m, float& sum) {
    m = -INFINITY;
#pragma unroll 1
    for (int j = 0; j < n; ++j) {
        const float x = y(j);
        if (x > m || x != x) m = x;
    }
    if (fabsf(m) == INFINITY) m = 0.f;
    sum = 0.f;
#pragma unroll 1
    for (int j = 0; j < n; ++j) sum = fadd(sum, expf(fsub(y(j), m)));
    return fadd(logf(sum), m);
}

template <int NT, int MODE>
__global__ void __launch_bounds__(NT) soft_td_fwd_kernel(SoftTdArgs a, float* ws) {
    pdl_prologue();
    constexpr int K = MODE == 0 ? 2 : 1;  // loss (and the action gap)
    __shared__ float s_coef[NT];
    __shared__ int s_act[NT];
    const long long r0 = (long long)blockIdx.x * NT;
    const long long r = r0 + threadIdx.x;
    const float inv_div = (float)(1.0 / a.loss_div);
    float acc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] = 0.f;
    s_coef[threadIdx.x] = 0.f;
    s_act[threadIdx.x] = -1;
    if (r < a.R) {
        const long long s = MODE == 2 ? r / a.G : r;  // G == 1 in modes 0 and 1
        const int N = a.N;
        const int act = (int)a.action[r];
        const float q_sa = a.q[r * N + act];
        const float nd = fsub(1.f, a.done[s]);
        float target;
        if (MODE == 0) {
            const float* __restrict__ tq = a.target_q + r * N;
            const float* __restrict__ nq = a.next_q + r * N;
            const float rw = a.reward[s];
            // row max of target_q (torch.max: NaN propagates) and its top two for the action gap (topk: equal maxima give 0,
            // NaN ranks above every number)
            float v = -INFINITY, t1 = -INFINITY, t2 = -INFINITY, vn = -INFINITY;
            for (int j = 0; j < N; ++j) {
                const float x = tq[j], y = nq[j];
                if (x > v || x != x) v = x;
                if (y > vn || y != y) vn = y;
                if (x > t1 || x != x) {
                    t2 = t1;
                    t1 = x;
                } else if (x > t2) {
                    t2 = x;
                }
            }
            float m, sm, mn, smn;
            const float lse = row_logsumexp([&](int j) { return __fdiv_rn(fsub(tq[j], v), a.tau); }, N, m, sm);
            const float lse_n = row_logsumexp([&](int j) { return __fdiv_rn(fsub(nq[j], vn), a.tau); }, N, mn, smn);
            const float lp = fsub(fsub(tq[act], v), fmul(a.tau, lse));  // log_pi.gather(1, act), td.py:132-135
            const float clamped = lp != lp ? lp : fminf(fmaxf(lp, -1.f), 1.f);  // torch.clamp keeps NaN
            a.clipfrac[r] = (lp > 1.f || lp < -1.f) ? 1.f : 0.f;
            const float tl = fmul(a.tau, lse_n);
            float soft = 0.f;  // sum_j pi'_j * (q'_j - tau_log_pi'_j) * (1 - d), td.py:141-145
            for (int j = 0; j < N; ++j) {
                const float d = fsub(nq[j], vn);
                const float pi = __fdiv_rn(expf(fsub(__fdiv_rn(d, a.tau), mn)), smn);
                soft = fadd(soft, fmul(fmul(pi, fsub(nq[j], fsub(d, tl))), nd));
            }
            target = fadd(fadd(rw, fmul(a.alpha, clamped)), fmul(a.gamma, soft));  // td.py:147
            acc[1] = fsub(t1, t2);
        } else if (MODE == 1) {
            const float* __restrict__ nq = a.next_q + r * N;
            const float* __restrict__ rw = a.reward + r;
            const size_t Bi = (size_t)a.R;
            float rwv[8];
            nstep_reward_load(rwv, rw, Bi, a.cum_reward ? 1 : a.nstep);
            const float vg = a.value_gamma ? a.value_gamma[r * a.value_gamma_stride] : a.gamma_pow_n;
            float ret;
            if (a.cum_reward) {
                ret = rwv[0];
            } else {
                float rf;
                ret = nstep_reward_sum(rwv, rw, Bi, a.nstep, a.gamma, rf);
            }
            float m, sm;
            float tv = fmul(a.alpha, row_logsumexp([&](int j) { return __fdiv_rn(nq[j], a.alpha); }, N, m, sm));
            if (tv == INFINITY) tv = 20.f;  // td.py:1230-1231; NaN stays NaN
            else if (tv == -INFINITY) tv = -20.f;
            if (a.record_v) a.record_v[r] = tv;
            target = fadd(ret, fmul(fmul(vg, tv), nd));  // td.py:1239 / :1241 / nstep_return :267, :273
        } else {
            target = fadd(fmul(fmul(a.gamma, nd), a.next_q[r]), a.reward[s]);  // td.py:205 / :217
        }
        const float w = a.weight ? a.weight[r] : 1.f;  // read after the target: one value fewer live across the row loops
        float dx;
        const float td = criterion_eval(a.criterion, a.crit_param, q_sa, target, dx);
        a.td_err[r] = td;
        if (a.target) a.target[r] = target;
        a.dcrit[r] = dx;
        acc[0] = td * w;
        if (a.grad_unit) {
            s_coef[threadIdx.x] = w * dx * inv_div;
            s_act[threadIdx.x] = act;
        }
    }
    if (a.grad_unit) store_onehot_rows<NT>(a.grad_unit, r0, a.R, a.N, s_coef, s_act);
    td_loss_sum<K, NT>(acc, ws, false, [&](int k, double t) {
        const float v = (float)(t / a.loss_div);
        if (k == 0) a.loss[0] = v;
        else a.action_gap[0] = v;
    });
}

// ---------------------------------------------------------------------------------------------------------------
// C51 categorical projection: one warp per (sample, agent) row, lanes stride the atoms, the projected distribution is
// accumulated with shared-memory atomics (the index_add_ of td.py:510-511) and kept for the backward pass.
// ---------------------------------------------------------------------------------------------------------------
struct DntdArgs {
    const float* dist;       // (R, N, n_atom)
    const float* next_dist;  // (R, N, n_atom)
    const long long* act;    // (R)
    const long long* next_act;
    const float* reward;  // (nstep, B)
    const float* done;    // (B)
    const float* weight;  // null, or stride 0 / 1 over R
    long long weight_stride;
    const float* value_gamma;  // null or stride 0 / 1 over B
    long long value_gamma_stride;
    const float* support;  // (n_atom), torch.linspace(v_min, v_max, n_atom) computed by the caller
    long long R;
    long long A;  // rows per batch entry (1 single agent)
    long long B;
    int N;
    int n_atom;
    int nstep;
    float gamma;
    float gamma_pow_n;
    float v_min, v_max, delta_z;
    float* loss;
    float* td_err;  // (R)
    float* proj;    // (R, n_atom)
    int* bad_flag;  // set to 1 if any selected dist entry is <= 0 (td.py:513)
    float* grad_unit;  // nullable (R, N, n_atom): d loss / d dist for a unit upstream gradient
};

// NJ = atoms per lane (ceil(n_atom / 32), 2 for C51): every global operand of a row -- the chosen rows of dist / next_n_dist,
// the support, the n-step rewards -- is requested in ONE batch right after the two action indices have arrived, and lives in
// registers from then on (reloading dist[j] in every iteration of the gradient loop costs 12 dependent L2 round trips per
// row).
template <int NT, int NJ>
__global__ void __launch_bounds__(NT) dntd_fwd_kernel(DntdArgs a, float* ws) {
    pdl_prologue();
    extern __shared__ float s_proj[];  // [NT/32][n_atom]
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long r = (long long)blockIdx.x * (NT / 32) + wid;
    const int na = a.n_atom;
    float* pj = s_proj + wid * na;
    float acc[1] = {0.f};
    // a row's work is one serial chain in one warp (~700 instructions): 32-bit index arithmetic; the bin positions keep the
    // IEEE division of td.py:500
    if (r < a.R) {
        const long long b = r / a.A;
        const int sel = (int)a.act[r], nsel = (int)a.next_act[r];
        const float* __restrict__ nd = a.next_dist + (r * a.N + nsel) * na;
        const float* __restrict__ dd = a.dist + (r * a.N + sel) * na;
        float p_[NJ], d_[NJ], z_[NJ];
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
            const int j = lane + 32 * u;
            const bool ok = j < na;
            p_[u] = ok ? nd[j] : 0.f;
            d_[u] = ok ? dd[j] : 1.f;
            z_[u] = ok ? a.support[j] : 0.f;
            if (ok) pj[j] = 0.f;
        }
        // every per-sample scalar is requested before any is used
        const float* __restrict__ rw = a.reward + b;
        const size_t Bi = (size_t)a.B;
        float rwv[8];
        nstep_reward_load(rwv, rw, Bi, a.nstep);
        const float dn = a.done[b];
        const float vg = a.value_gamma ? a.value_gamma[b * a.value_gamma_stride] : a.gamma_pow_n;
        const float w = a.weight ? a.weight[r * a.weight_stride] : 1.f;
        float rf;
        const float ret = nstep_reward_sum(rwv, rw, Bi, a.nstep, a.gamma, rf);
        const float scale = fmul(fsub(1.f, dn), vg);  // (1-done) * gamma**n, td.py:492-498
        __syncwarp();
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
            const int j = lane + 32 * u;
            int key = -1 - lane;  // lanes past n_atom: unique keys, zero contributions
            float clo = 0.f, chi = 0.f;
            if (j < na) {
                float tz = fadd(ret, fmul(scale, z_[u]));
                tz = fminf(fmaxf(tz, a.v_min), a.v_max);
                const float pos = __fdiv_rn(fsub(tz, a.v_min), a.delta_z);  // td.py:500
                float lo = floorf(pos), hi = ceilf(pos);
                if (hi > 0.f && lo == hi) lo -= 1.f;                          // td.py:504
                if (lo < (float)(na - 1) && lo == hi) hi += 1.f;              // td.py:505 (now hi == lo + 1 always)
                key = (int)lo;
                clo = fmul(p_[u], fsub(hi, pos));
                chi = fmul(p_[u], fsub(pos, lo));
            }
            // Tz is monotone in the atom index, so lanes that hit the same bin are CONTIGUOUS (a terminal sample, done = 1, or a
            // clamped tail sends all of them to one bin): a segmented warp scan adds them up and only the last lane of a
            // segment touches shared memory instead of 32 lanes contending in a CAS loop on one word
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int k2 = __shfl_up_sync(0xffffffffu, key, d);
                const float l2 = __shfl_up_sync(0xffffffffu, clo, d), h2 = __shfl_up_sync(0xffffffffu, chi, d);
                if (lane >= d && k2 == key) {
                    clo += l2;
                    chi += h2;
                }
            }
            const int knext = __shfl_down_sync(0xffffffffu, key, 1);
            if (key >= 0 && (lane == 31 || knext != key)) {
                atomicAdd(&pj[key], clo);
                atomicAdd(&pj[key + 1], chi);
            }
        }
        __syncwarp();
        float td = 0.f;
        bool bad = false;
        float m_[NJ];
        float* __restrict__ prow = a.proj + r * na;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
            const int j = lane + 32 * u;
            m_[u] = 0.f;
            if (j < na) {
                m_[u] = pj[j];
                bad |= !(d_[u] > 0.f);
                // IEEE logf: the MUFU lg2 flushes a subnormal probability to -inf (NaN against zero mass) and is off by
                // ~2^-22 near 1, i.e. by percents on the TD error of a near-converged row
                td = fmaf(logf(d_[u]), m_[u], td);
                prow[j] = m_[u];
            }
        }
        td = -warp_sum(td);
        if (a.bad_flag && __any_sync(0xffffffffu, bad) && lane == 0) atomicOr(a.bad_flag, 1);
        if (lane == 0) {
            a.td_err[r] = td;
            acc[0] = td * w;
        }
        if (a.grad_unit) {  // dense (N, n_atom) gradient block of the row: non-zero on the chosen action only
            const float c = -w / (float)a.R;
            float* __restrict__ gr = a.grad_unit + r * a.N * na;
            float g_[NJ];
#pragma unroll
            for (int u = 0; u < NJ; ++u) g_[u] = __fdiv_rn(c * m_[u], d_[u]);  // IEEE division, as dntd_bwd_kernel
            const int Ni = a.N;
            for (int n = 0; n < Ni; ++n) {
#pragma unroll
                for (int u = 0; u < NJ; ++u) {
                    const int j = lane + 32 * u;
                    if (j < na) gr[n * na + j] = (n == sel) ? g_[u] : 0.f;
                }
            }
        }
    }
    td_loss_sum<1, NT>(acc, ws, false, [&](int, double t) { a.loss[0] = (float)(t / (double)a.R); });
}

__global__ void dntd_bwd_kernel(const float* __restrict__ dist, const long long* __restrict__ act,
                                const float* __restrict__ proj, const float* __restrict__ weight,
                                long long weight_stride, const float* __restrict__ g_loss,
                                const float* __restrict__ g_td, long long R, int N, int n_atom, int skip_if_unit,
                                float* __restrict__ grad_dist) {
    pdl_prologue();
    // skip_if_unit: the forward launch already wrote grad_dist for a unit upstream gradient -- verify and leave
    if (skip_if_unit && !g_td && g_loss && *g_loss == 1.f) return;
    const long long per_row = (long long)N * n_atom;
    const float g = g_loss ? *g_loss : 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < R * per_row;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / per_row;
        const int rem = (int)(i - r * per_row);
        const int n = rem / n_atom, j = rem - n * n_atom;
        float out = 0.f;
        if (n == (int)act[r]) {
            const float w = weight ? weight[r * weight_stride] : 1.f;
            float c = g * w / (float)R;
            if (g_td) c += g_td[r];  // the unweighted per-sample error carries gradient too (td.py:519)
            out = -c * proj[r * n_atom + j] / dist[i];
        }
        grad_dist[i] = out;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// lambda-return scan along T on a (T, B) tile -- same three-phase tile scheme as gae.cu.
//   G_{T-1} = r + ((1-d)*gamma)*V_T ;  G_t = r_t + (1-d_t)*(disc_t*G_{t+1} + (gamma_t - disc_t)*V_{t+1}),  disc = gamma*lambda
// MODE 0: gamma/lambda scalars or (T,B) tensors, optional done (generalized_lambda_returns, td.py:1574-1651)
// MODE 1: UPGO: gamma = 1, lambda_t = [r_{t+1} + V_{t+2} >= V_{t+1}], last = 1 (upgo.py:66-68)
// HEAD 1: fused TD(lambda) loss head: loss = 0.5*mean(w*(G - V_t)^2) and the saved gradient dV (td.py:1570)
// HEAD 2: COMA's value loss (coma.py:45-52), on ComaLamArgs: column c = b*A + a of a (T-1, B*A) scan whose bootstrap values
//         are target_q_value[t, b, a, action[t, b, a]] and whose reward is reward[t, b], both read in place (no gathered or
//         broadcast copy); loss = mean(w*(G - q_taken)^2) over rows t < T-1, and the saved unit gradient of each column
// ---------------------------------------------------------------------------------------------------------------
struct LamArgs {
    const float* value;   // (T+1, B)
    const float* reward;  // (T, B)
    const float* gammas;  // nullable (T, B)
    const float* lambdas; // nullable (T, B)
    const float* done;    // nullable (T, B)
    const float* weight;  // HEAD: nullable (T, B)
    float gamma, lambda;
    long long T, B;
    float* ret;     // (T, B) output (nullable when HEAD)
    float* loss;    // HEAD
    float* dvalue;  // HEAD: (T+1, B) saved d loss / d value for unit upstream gradient
};

// HEAD 2's operands.  The scan runs over T = T_coma - 1 rows and B = B_coma * A columns; value is unused.
struct ComaLamArgs : LamArgs {
    const long long* action;  // (T+1, B)
    const float* target_q;    // (T+1, B, N)
    const float* q;           // (T+1, B, N)
    long long A;              // agents: reward column of scan column c is c / A
    int N;
    float* dq;    // (T, B) d loss / d q_value[t, b, a, action] for a unit upstream gradient
    float* dret;  // nullable (T, B): d loss / d G, for callers that differentiate the returns
};

template <int TC, int NT, int CHUNK, int MODE, int HEAD, class Args>
__device__ __forceinline__ void lambda_scan(const Args& a, float* ws) {
    // Chunks of CHUNK time steps, newest first, double-buffered: while the TC scan lanes run the dependent chain of chunk k
    // out of shared memory, every thread already has the global loads of chunk k+1 in flight (U elements per thread in
    // registers); they are turned into the scan's operands and written to the other buffer once the scan is done.  (Without
    // the overlap a long T pays load latency + scan + store in a row for every chunk.)
    constexpr int U = CHUNK * TC / NT;
    static_assert(U * NT == CHUNK * TC && U >= 1, "one pass per chunk");
    __shared__ float s_r[2][CHUNK][TC];
    __shared__ float s_m[2][CHUNK][TC];
    __shared__ float s_disc[2][CHUNK][TC];
    __shared__ float s_c[2][CHUNK][TC];
    // HEAD: V_t and the weight of the chunk, fetched with the scan operands one chunk ahead (single-buffered: a thread writes
    // the slots of chunk k+1 only after it has consumed the same slots of chunk k)
    __shared__ float s_hv[HEAD ? CHUNK : 1][TC];
    __shared__ float s_hw[HEAD ? CHUNK : 1][TC];
    const long long c0 = (long long)blockIdx.x * TC;
    const long long T = a.T, B = a.B;
    struct Raw {
        float rw[U], vn[U], g[U], l[U], dn[U], r2[U], v2[U], hv[U], hw[U];
        bool ok[U];
    };
    // all global loads of a chunk are issued before any of them is consumed
    auto fetch = [&](long long lo, int rows, Raw& x) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = threadIdx.x + u * NT;
            const int r = i / TC, cc = i % TC;
            const long long c = c0 + cc, t = lo + r;
            x.ok[u] = i < rows * TC && c < B;
            x.rw[u] = x.vn[u] = x.dn[u] = x.r2[u] = x.v2[u] = 0.f;
            x.g[u] = a.gamma;
            x.l[u] = a.lambda;
            if (x.ok[u]) {
                const long long off = t * B + c;
                if constexpr (HEAD == 2) {
                    const long long nx = off + B;  // (t+1, c): the bootstrap value gathered through the action index
                    x.rw[u] = a.reward[t * (B / a.A) + c / a.A];
                    x.vn[u] = a.target_q[nx * a.N + a.action[nx]];
                    x.hv[u] = a.q[off * a.N + a.action[off]];
                    x.hw[u] = a.weight ? a.weight[off] : 1.f;
                    continue;
                } else {
                    x.rw[u] = a.reward[off];
                    x.vn[u] = a.value[off + B];  // V_{t+1}
                }
                if (MODE == 1) {
                    if (t < T - 1) {
                        x.r2[u] = a.reward[off + B];
                        x.v2[u] = a.value[off + 2 * B];
                    }
                } else {
                    if (a.gammas) x.g[u] = a.gammas[off];
                    if (a.lambdas) x.l[u] = a.lambdas[off];
                }
                if (a.done) x.dn[u] = a.done[off];
                if (HEAD == 1) {
                    x.hv[u] = a.value[off];
                    x.hw[u] = a.weight ? a.weight[off] : 1.f;
                }
            }
        }
    };
    auto commit = [&](int buf, long long lo, const Raw& x) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (!x.ok[u]) continue;
            const int i = threadIdx.x + u * NT;
            const int r = i / TC, cc = i % TC;
            const long long t = lo + r;
            float gg = x.g[u], ll = x.l[u];
            if (MODE == 1) {
                gg = 1.f;
                ll = 1.f;
                if (t < T - 1) ll = (fadd(x.r2[u], x.v2[u]) >= x.vn[u]) ? 1.f : 0.f;
            }
            const float m = a.done ? fsub(1.f, x.dn[u]) : 1.f;
            const float disc = fmul(gg, ll);
            if (HEAD != 0) {
                s_hv[r][cc] = x.hv[u];
                s_hw[r][cc] = x.hw[u];
            }
            s_r[buf][r][cc] = x.rw[u];
            s_m[buf][r][cc] = m;
            if (t == T - 1) {
                // closed form of the last row kept in s_c; disc = 0 so the carry (0) is ignored exactly
                s_disc[buf][r][cc] = 0.f;
                s_c[buf][r][cc] = fmul(fmul(m, gg), x.vn[u]);
                s_m[buf][r][cc] = 1.f;
            } else {
                s_disc[buf][r][cc] = disc;
                s_c[buf][r][cc] = fmul(fsub(gg, disc), x.vn[u]);
            }
        }
    };
    float carry = 0.f;
    float acc[1] = {0.f};
    {
        const long long lo = T > CHUNK ? T - CHUNK : 0;
        Raw x;
        fetch(lo, (int)(T - lo), x);
        commit(0, lo, x);
    }
    __syncthreads();
    int buf = 0;
    for (long long hi = T; hi > 0; hi -= CHUNK, buf ^= 1) {
        const long long lo = hi > CHUNK ? hi - CHUNK : 0;
        const int rows = (int)(hi - lo);
        const bool have_next = lo > 0;
        const long long nlo = lo > CHUNK ? lo - CHUNK : 0;
        Raw nx;
        if (have_next) fetch(nlo, (int)(lo - nlo), nx);
        if (threadIdx.x < TC && c0 + threadIdx.x < B) {
            const int cc = threadIdx.x;
            // 16 rows at a time: the shared-memory operands of the next 16 steps are in registers before the dependent
            // chain needs them, so each step costs only its 4 dependent fp32 operations
            constexpr int UU = 16;
            int r = rows - 1;
            for (; r >= UU - 1; r -= UU) {
                float rr[UU], mm[UU], dd[UU], cq[UU];
#pragma unroll
                for (int j = 0; j < UU; ++j) {
                    rr[j] = s_r[buf][r - j][cc];
                    mm[j] = s_m[buf][r - j][cc];
                    dd[j] = s_disc[buf][r - j][cc];
                    cq[j] = s_c[buf][r - j][cc];
                }
#pragma unroll
                for (int j = 0; j < UU; ++j) {
                    carry = fadd(rr[j], fmul(mm[j], fadd(fmul(dd[j], carry), cq[j])));
                    s_r[buf][r - j][cc] = carry;
                }
            }
            for (; r >= 0; --r) {
                carry = fadd(s_r[buf][r][cc], fmul(s_m[buf][r][cc], fadd(fmul(s_disc[buf][r][cc], carry), s_c[buf][r][cc])));
                s_r[buf][r][cc] = carry;
            }
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = threadIdx.x + u * NT;
            const int r = i / TC, cc = i % TC;
            if (i >= rows * TC || c0 + cc >= B) continue;
            const long long off = (lo + r) * B + c0 + cc;
            const float gret = s_r[buf][r][cc];
            if (a.ret) a.ret[off] = gret;
            if (HEAD == 1) {
                const float w = s_hw[r][cc];
                const float d = gret - s_hv[r][cc];
                acc[0] += w * d * d;
                a.dvalue[off] = -w * d / (float)(T * B);  // 0.5 * w * 2 * (V - G) / count
            }
            if constexpr (HEAD == 2) {
                const float w = s_hw[r][cc];
                const float d = gret - s_hv[r][cc];
                acc[0] += w * d * d;
                const float g = 2.f * w * d / (float)(T * B);  // w * 2 * (G - q) / count
                a.dq[off] = -g;
                if (a.dret) a.dret[off] = g;
            }
        }
        if (have_next) commit(buf ^ 1, nlo, nx);
        __syncthreads();
    }
    if (HEAD == 1) {
        // last value row receives no gradient (value[:-1], td.py:1570)
        for (int cc = threadIdx.x; cc < TC; cc += NT)
            if (c0 + cc < B) a.dvalue[T * B + c0 + cc] = 0.f;
        double tot[1];
        if (grid_sum<1, NT>(acc, tot, ws, 0) && threadIdx.x == 0)
            a.loss[0] = (float)(0.5 * tot[0] / ((double)T * (double)B));
    }
    if constexpr (HEAD == 2) {
        double tot[1];
        if (grid_sum<1, NT>(acc, tot, ws, 0) && threadIdx.x == 0) a.loss[0] = (float)(tot[0] / ((double)T * (double)B));
    }
}

template <int TC, int NT, int CHUNK, int MODE, int HEAD>
__global__ void __launch_bounds__(NT) lambda_scan_kernel(LamArgs a, float* ws) {
    pdl_prologue();
    lambda_scan<TC, NT, CHUNK, MODE, HEAD>(a, ws);
}

template <int TC, int NT, int CHUNK>
__global__ void __launch_bounds__(NT) lambda_scan_coma_kernel(ComaLamArgs a, float* ws) {
    pdl_prologue();
    lambda_scan<TC, NT, CHUNK, 0, 2>(a, ws);
}

// Backward of the lambda-return scan (generalized_lambda_returns is differentiable in the reference, td.py:1574-1651; MBSAC
// and Dreamer back-propagate an actor loss through it): the transposed recurrence runs FORWARD in time,
//   a_t = gG_t + (1-d_{t-1})*disc_{t-1}*a_{t-1};  dr_t = a_t;  dV_{t+1} = a_t*(1-d_t)*(gamma_t - disc_t)  (last row: gamma_t)
// and, when the (T, B) gamma / lambda tensors want gradients, dgamma_t = a_t*(1-d_t)*(lambda_t*G_{t+1} + (1-lambda_t)*V_{t+1}),
// dlambda_t = a_t*(1-d_t)*gamma_t*(G_{t+1} - V_{t+1}).  Thread = column; every load of a step is independent of the carry.
struct LamBwdArgs {
    const float* g_ret;    // (T, B) upstream gradient
    const float* value;    // (T+1, B)
    const float* reward;   // (T, B)  (upgo mode: drives lambda)
    const float* ret;      // (T, B) forward result (needed for dgamma / dlambda only)
    const float* gammas;   // nullable
    const float* lambdas;  // nullable
    const float* done;     // nullable
    float gamma, lambda;
    int upgo_mode;
    long long T, B;
    float* g_value;    // (T+1, B)
    float* g_reward;   // nullable (T, B)
    float* g_gammas;   // nullable (T, B)
    float* g_lambdas;  // nullable (T, B)
};

template <int NT>
__global__ void __launch_bounds__(NT) lambda_returns_bwd_kernel(LamBwdArgs a) {
    pdl_prologue();
    const long long c = (long long)blockIdx.x * NT + threadIdx.x;
    if (c >= a.B) return;
    const long long T = a.T, B = a.B;
    a.g_value[c] = 0.f;
    float adj = 0.f, coef = 0.f;
    constexpr int U = 8;
    for (long long t0 = 0; t0 < T; t0 += U) {
        float g[U], gg[U], ll[U], m[U], vn[U], gn[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {  // all loads of U steps first
            const long long t = t0 + u;
            g[u] = 0.f; gg[u] = a.gamma; ll[u] = a.lambda; m[u] = 1.f; vn[u] = 0.f; gn[u] = 0.f;
            if (t < T) {
                const long long off = t * B + c;
                g[u] = a.g_ret[off];
                if (a.upgo_mode) {
                    gg[u] = 1.f;
                    ll[u] = 1.f;
                    if (t < T - 1) ll[u] = (fadd(a.reward[off + B], a.value[off + 2 * B]) >= a.value[off + B]) ? 1.f : 0.f;
                } else {
                    if (a.gammas) gg[u] = a.gammas[off];
                    if (a.lambdas) ll[u] = a.lambdas[off];
                }
                if (a.done) m[u] = 1.f - a.done[off];
                if (a.g_gammas || a.g_lambdas) {
                    vn[u] = a.value[off + B];
                    gn[u] = (t < T - 1) ? a.ret[off + B] : 0.f;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long t = t0 + u;
            if (t >= T) break;
            const long long off = t * B + c;
            adj = fmaf(coef, adj, g[u]);
            if (a.g_reward) a.g_reward[off] = adj;
            const float am = adj * m[u];
            if (t == T - 1) {
                a.g_value[off + B] = am * gg[u];
                if (a.g_gammas) a.g_gammas[off] = am * vn[u];
                if (a.g_lambdas) a.g_lambdas[off] = 0.f;
            } else {
                const float disc = gg[u] * ll[u];
                a.g_value[off + B] = am * (gg[u] - disc);
                if (a.g_gammas) a.g_gammas[off] = am * (ll[u] * gn[u] + (1.f - ll[u]) * vn[u]);
                if (a.g_lambdas) a.g_lambdas[off] = am * gg[u] * (gn[u] - vn[u]);
                coef = m[u] * disc;
            }
        }
    }
}

// out[i] = (*g) * in[i]  -- backward of the heads that saved their unit-upstream gradient in the forward pass
__global__ void scale_kernel(const float* __restrict__ g, const float* __restrict__ in, float* __restrict__ out,
                             long long n) {
    pdl_prologue();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (*g) * in[i];
}

}  // namespace b200rl

using namespace b200rl;

static double qntd_loss_div(long long S, long long G, long long seq_len) {
    if (seq_len <= 0) return (double)S * (double)G;  // (td * weight).mean() over every row
    // sequence form: sum_t mean_b(...) / (len + 1e-8) -- a python float that torch narrows to fp32 (r2d2.py:364)
    return (double)(S / seq_len) * (double)G * (double)(float)((double)seq_len + 1e-8);
}

// python's `gamma ** nstep`: libm pow in double, then fp32
static float gamma_pow(double gamma, int nstep) { return (float)pow(gamma, (double)nstep); }

static TdScalars td_scalars(double gamma, int nstep, double rescale_eps, long long S, long long G, long long seq_len,
                            double priority_mix) {
    TdScalars c{};
    c.gamma = (float)gamma;
    c.gamma_pow_n = gamma_pow(gamma, nstep);
    c.eps = (float)rescale_eps; c.four_eps = (float)(4.0 * rescale_eps); c.two_eps = (float)(2.0 * rescale_eps);
    c.loss_div = qntd_loss_div(S, G, seq_len);
    c.prio_max_w = (float)priority_mix; c.prio_mean_w = (float)(1.0 - priority_mix);
    c.prio_div = (float)((double)seq_len + 1e-8);
    return c;
}

extern "C" int b200rl_qntd_fwd(const float* q, const float* next_n_q, const long long* action,
                               const long long* next_n_action, const float* reward, const float* done,
                               const float* weight, const float* value_gamma, long long value_gamma_stride,
                               const float* gamma_per_sample, long long S, long long G, long long N, int nstep,
                               double gamma, int cum_reward, int rescale, double rescale_eps, int criterion,
                               double criterion_param, int group_mean, long long seq_len, double priority_mix,
                               float* loss, float* td_error_per_sample, float* dcrit_saved, float* target_out,
                               float* grad_q_unit, float* priority_out, float* workspace, size_t workspace_bytes,
                               void* stream) {
    if (S <= 0 || G < 1 || N < 1 || nstep < 1 || !q || !next_n_q || !action || !next_n_action || !reward || !done ||
        !loss || !td_error_per_sample || !dcrit_saved || !workspace)
        return B200RL_ERR_ARG;
    if (criterion < 0 || criterion > 3) return B200RL_ERR_ARG;
    if (seq_len < 0 || (seq_len > 0 && (S % seq_len != 0 || cum_reward)) || (priority_out && seq_len <= 0) ||
        (priority_out && (G != 1 || group_mean)))
        return B200RL_ERR_ARG;
    QntdArgs a{td_scalars(gamma, nstep, rescale_eps, S, G, seq_len, priority_mix)};
    a.q = q; a.next_q = next_n_q; a.action = action; a.next_action = next_n_action; a.reward = reward; a.done = done;
    a.weight = weight; a.value_gamma = value_gamma; a.value_gamma_stride = value_gamma_stride;
    a.gamma_ps = gamma_per_sample; a.S = S; a.Bcol = seq_len > 0 ? S / seq_len : S; a.G = (int)G; a.N = (int)N;
    a.nstep = nstep; a.cum_reward = cum_reward; a.rescale = rescale;
    a.criterion = criterion; a.crit_param = (float)criterion_param; a.group_mean = group_mean;
    a.loss = loss; a.td_err = td_error_per_sample; a.dcrit = dcrit_saved; a.target = target_out;
    a.grad_unit = grad_q_unit; a.priority = priority_out;
    return launch_td_rows<1>([](auto nt) { return qntd_fwd_kernel<decltype(nt)::value>; }, a, S, priority_out, workspace,
                             workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200rl_qntd_bwd(const float* dcrit_saved, const float* weight, const long long* action,
                               const float* g_loss, const float* g_td, long long S, long long G, long long N,
                               int group_mean, long long seq_len, int skip_if_unit, float* grad_q, void* stream) {
    if (S <= 0 || G < 1 || N < 1 || !dcrit_saved || !action || !grad_q) return B200RL_ERR_ARG;
    long long grid = div_up(S * G * N, 256);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;  // grid-stride; the verification launch normally returns at once
    const float inv_div = (float)(1.0 / qntd_loss_div(S, G, seq_len));
    return launch_k(qntd_bwd_kernel, (int)grid, 256, 0, (cudaStream_t)stream, dcrit_saved, weight, action, g_loss, g_td, S,
                    (int)G, (int)N, group_mean, inv_div, skip_if_unit, grad_q);
}

extern "C" int b200rl_dqfd_fwd(const float* q, const float* next_n_q, const float* new_n_q_one_step, const long long* action,
                               const long long* next_n_action, const long long* next_n_action_one_step, const float* reward,
                               const float* done, const float* done_one_step, const float* weight, const float* value_gamma,
                               long long value_gamma_stride, const float* is_expert, long long S, long long N, int nstep,
                               double gamma, int cum_reward, int rescale, double rescale_eps, int criterion,
                               double criterion_param, double lambda_n_step_td, double lambda_one_step_td,
                               double lambda_supervised_loss, double margin, long long seq_len, double priority_mix,
                               float* loss, float* td_error_per_sample, float* loss_statistics, float* saved,
                               float* target_n_out, float* target_1_out, float* grad_q_unit, float* priority_out,
                               float* workspace, size_t workspace_bytes, void* stream) {
    if (S <= 0 || N < 1 || N >= (1 << 24) || nstep < 1 || !q || !next_n_q || !new_n_q_one_step || !action ||
        !next_n_action || !next_n_action_one_step || !reward || !done || !done_one_step || !is_expert || !loss ||
        !td_error_per_sample || !loss_statistics || !saved || !workspace)
        return B200RL_ERR_ARG;
    if (criterion < -1 || criterion > 3) return B200RL_ERR_ARG;
    if (seq_len < 0 || (seq_len > 0 && (S % seq_len != 0 || cum_reward)) || (priority_out && seq_len <= 0))
        return B200RL_ERR_ARG;
    // a workspace under WS_MIN_BYTES is reported before a misaligned `saved`
    if (workspace_bytes >= WS_MIN_BYTES && reinterpret_cast<uintptr_t>(saved) % 16 != 0) return B200RL_ERR_ARG;
    DqfdArgs a{td_scalars(gamma, nstep, rescale_eps, S, 1, seq_len, priority_mix)};
    a.q = q; a.next_q = next_n_q; a.next_q1 = new_n_q_one_step; a.action = action; a.next_action = next_n_action;
    a.next_action1 = next_n_action_one_step; a.reward = reward; a.done = done; a.done1 = done_one_step; a.weight = weight;
    a.value_gamma = value_gamma; a.value_gamma_stride = value_gamma_stride; a.is_expert = is_expert;
    a.S = S; a.Bcol = seq_len > 0 ? S / seq_len : S; a.N = (int)N; a.nstep = nstep;
    a.cum_reward = cum_reward; a.rescale = rescale; a.criterion = criterion; a.crit_param = (float)criterion_param;
    a.lam_n = (float)lambda_n_step_td; a.lam_1 = (float)lambda_one_step_td; a.lam_s = (float)lambda_supervised_loss;
    a.margin = (float)margin;
    a.loss = loss; a.td_err = td_error_per_sample; a.stats = loss_statistics; a.saved = reinterpret_cast<float4*>(saved);
    a.target_n = target_n_out; a.target_1 = target_1_out; a.grad_unit = grad_q_unit; a.priority = priority_out;
    return launch_td_rows<4>([](auto nt) { return dqfd_fwd_kernel<decltype(nt)::value>; }, a, S, priority_out, workspace,
                             workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200rl_dqfd_bwd(const float* saved, const float* weight, const long long* action, const float* g_loss,
                               const float* g_td, const float* g_loss_statistics_n, const float* g_loss_statistics_1,
                               const float* g_loss_statistics_je, long long S, long long N, double lambda_n_step_td,
                               double lambda_one_step_td, double lambda_supervised_loss, long long seq_len, int skip_if_unit,
                               float* grad_q, void* stream) {
    if (S <= 0 || N < 1 || N >= (1 << 24) || seq_len < 0 || (seq_len > 0 && S % seq_len != 0) || !saved || !action ||
        !grad_q || reinterpret_cast<uintptr_t>(saved) % 16 != 0)
        return B200RL_ERR_ARG;
    long long grid = div_up(S * N, 256);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;  // grid-stride; the verification launch normally returns at once
    const float inv_div = (float)(1.0 / qntd_loss_div(S, 1, seq_len));
    return launch_k(dqfd_bwd_kernel, (int)grid, 256, 0, (cudaStream_t)stream, reinterpret_cast<const float4*>(saved), weight,
                    action, g_loss, g_td, g_loss_statistics_n, g_loss_statistics_1, g_loss_statistics_je, S, (int)N,
                    (float)lambda_n_step_td, (float)lambda_one_step_td, (float)lambda_supervised_loss, inv_div, skip_if_unit,
                    grad_q);
}

extern "C" int b200rl_soft_td_fwd(int mode, const float* q, const float* target_q, const float* next_q,
                                  const long long* action, const float* reward, const float* done, const float* weight,
                                  const float* value_gamma, long long value_gamma_stride, long long S, long long G,
                                  long long N, int nstep, double gamma, double tau, double alpha, int cum_reward,
                                  int criterion, double criterion_param, float* loss, float* td_error_per_sample,
                                  float* dcrit_saved, float* target_out, float* grad_q_unit, float* action_gap,
                                  float* clipfrac, float* record_target_v, float* workspace, size_t workspace_bytes,
                                  void* stream) {
    if (mode < 0 || mode > 2 || S <= 0 || G < 1 || N < 1 || !q || !next_q || !action || !reward || !done || !loss ||
        !td_error_per_sample || !dcrit_saved || !workspace)
        return B200RL_ERR_ARG;
    if (criterion < 0 || criterion > 3) return B200RL_ERR_ARG;
    if (mode != 2 && G != 1) return B200RL_ERR_ARG;
    if (mode == 0 && (N < 2 || !target_q || !action_gap || !clipfrac)) return B200RL_ERR_ARG;
    if (mode == 1 && nstep < 1) return B200RL_ERR_ARG;
    if (mode != 1 && (cum_reward || value_gamma)) return B200RL_ERR_ARG;
    if (mode != 1) nstep = 1;
    SoftTdArgs a{td_scalars(gamma, nstep, 0.0, S, G, 0, 0.0)};
    a.q = q; a.target_q = target_q; a.next_q = next_q; a.action = action; a.reward = reward; a.done = done;
    a.weight = weight; a.value_gamma = value_gamma; a.value_gamma_stride = value_gamma_stride;
    a.R = S * G; a.G = (int)G; a.N = (int)N; a.nstep = nstep;
    a.tau = (float)tau; a.alpha = (float)alpha; a.cum_reward = cum_reward;
    a.criterion = criterion; a.crit_param = (float)criterion_param;
    a.loss = loss; a.td_err = td_error_per_sample; a.dcrit = dcrit_saved; a.target = target_out; a.grad_unit = grad_q_unit;
    a.action_gap = action_gap; a.clipfrac = clipfrac; a.record_v = record_target_v;
    const cudaStream_t st = (cudaStream_t)stream;
    if (mode == 0)
        return launch_td_rows<2>([](auto nt) { return soft_td_fwd_kernel<decltype(nt)::value, 0>; }, a, a.R, false, workspace,
                                 workspace_bytes, st);
    if (mode == 1)
        return launch_td_rows<1>([](auto nt) { return soft_td_fwd_kernel<decltype(nt)::value, 1>; }, a, a.R, false, workspace,
                                 workspace_bytes, st);
    return launch_td_rows<1>([](auto nt) { return soft_td_fwd_kernel<decltype(nt)::value, 2>; }, a, a.R, false, workspace,
                             workspace_bytes, st);
}

extern "C" int b200rl_dntd_fwd(const float* dist, const float* next_n_dist, const long long* act,
                               const long long* next_n_act, const float* reward, const float* done,
                               const float* weight, long long weight_stride, const float* value_gamma,
                               long long value_gamma_stride, const float* support, long long B, long long A,
                               long long N, int n_atom, int nstep, double gamma, double v_min, double v_max,
                               float* loss, float* td_error_per_sample, float* proj_saved, int* bad_flag,
                               float* grad_dist_unit, float* workspace, size_t workspace_bytes, void* stream) {
    if (B <= 0 || A < 1 || N < 1 || n_atom < 2 || nstep < 1 || !dist || !next_n_dist || !act || !next_n_act ||
        !reward || !done || !support || !loss || !td_error_per_sample || !proj_saved || !workspace)
        return B200RL_ERR_ARG;
    DntdArgs a{};
    a.dist = dist; a.next_dist = next_n_dist; a.act = act; a.next_act = next_n_act; a.reward = reward; a.done = done;
    a.weight = weight; a.weight_stride = weight_stride; a.value_gamma = value_gamma;
    a.value_gamma_stride = value_gamma_stride; a.support = support; a.R = B * A; a.A = A; a.B = B; a.N = (int)N;
    a.n_atom = n_atom; a.nstep = nstep; a.gamma = (float)gamma; a.gamma_pow_n = gamma_pow(gamma, nstep);
    a.v_min = (float)v_min; a.v_max = (float)v_max; a.delta_z = (float)((v_max - v_min) / (double)(n_atom - 1));
    a.loss = loss; a.td_err = td_error_per_sample; a.proj = proj_saved; a.bad_flag = bad_flag;
    a.grad_unit = grad_dist_unit;
    if (workspace_bytes < WS_MIN_BYTES) return B200RL_ERR_WORKSPACE;
    if (n_atom > 256) return B200RL_ERR_ARG;  // 8 atoms per lane in registers
    cudaStream_t st = (cudaStream_t)stream;
    if (a.R <= 8 * 511) {  // 8 rows per CTA: few enough CTAs for the one-round-trip reduction
        constexpr int NT = 256;
        const size_t sm = (size_t)(NT / 32) * n_atom * sizeof(float);
        const int grid = div_up(a.R, NT / 32);
        if (n_atom <= 64) return launch_k(dntd_fwd_kernel<NT, 2>, grid, NT, sm, st, a, workspace);
        return launch_k(dntd_fwd_kernel<NT, 8>, grid, NT, sm, st, a, workspace);
    }
    constexpr int NT = 128;
    const int grid = div_up(a.R, NT / 32);
    if ((size_t)(WS_CTRL_WORDS + grid) > WS_PARTIAL_LIMIT_WORDS) return B200RL_ERR_WORKSPACE;
    const size_t sm = (size_t)(NT / 32) * n_atom * sizeof(float);
    if (n_atom <= 64) return launch_k(dntd_fwd_kernel<NT, 2>, grid, NT, sm, st, a, workspace);
    return launch_k(dntd_fwd_kernel<NT, 8>, grid, NT, sm, st, a, workspace);
}

extern "C" int b200rl_dntd_bwd(const float* dist, const long long* act, const float* proj_saved, const float* weight,
                               long long weight_stride, const float* g_loss, const float* g_td, long long R,
                               long long N, int n_atom, int skip_if_unit, float* grad_dist, void* stream) {
    if (R <= 0 || N < 1 || n_atom < 2 || !dist || !act || !proj_saved || !grad_dist) return B200RL_ERR_ARG;
    long long grid = div_up(R * N * n_atom, 256);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;  // grid-stride; the verification launch normally returns at once
    return launch_k(dntd_bwd_kernel, (int)grid, 256, 0, (cudaStream_t)stream, dist, act, proj_saved, weight, weight_stride, g_loss, g_td,
                    R, (int)N, n_atom, skip_if_unit, grad_dist);
}

template <int MODE, int HEAD>
static int launch_lambda(const LamArgs& a, float* ws, cudaStream_t st) {
    if (a.B >= 16 * 2 * NUM_SMS) return launch_k(lambda_scan_kernel<16, 256, 64, MODE, HEAD>, div_up(a.B, 16), 256, 0, st, a, ws);
    return launch_k(lambda_scan_kernel<8, 256, 128, MODE, HEAD>, div_up(a.B, 8), 256, 0, st, a, ws);
}

extern "C" int b200rl_lambda_returns(const float* value, const float* reward, const float* gammas, double gamma,
                                     const float* lambdas, double lambda_, const float* done, int upgo_mode,
                                     long long T, long long B, float* ret, void* stream) {
    if (T <= 0 || B <= 0 || !value || !reward || !ret) return B200RL_ERR_ARG;
    LamArgs a{};
    a.value = value; a.reward = reward; a.gammas = gammas; a.lambdas = lambdas; a.done = done;
    a.gamma = (float)gamma; a.lambda = (float)lambda_; a.T = T; a.B = B; a.ret = ret;
    return upgo_mode ? launch_lambda<1, 0>(a, nullptr, (cudaStream_t)stream)
                     : launch_lambda<0, 0>(a, nullptr, (cudaStream_t)stream);
}

extern "C" int b200rl_lambda_returns_bwd(const float* g_ret, const float* value, const float* reward, const float* ret,
                                         const float* gammas, double gamma, const float* lambdas, double lambda_,
                                         const float* done, int upgo_mode, long long T, long long B, float* grad_value,
                                         float* grad_reward, float* grad_gammas, float* grad_lambdas, void* stream) {
    if (T <= 0 || B <= 0 || !g_ret || !value || !grad_value) return B200RL_ERR_ARG;
    if ((upgo_mode && !reward) || ((grad_gammas || grad_lambdas) && !ret)) return B200RL_ERR_ARG;
    LamBwdArgs a{};
    a.g_ret = g_ret; a.value = value; a.reward = reward; a.ret = ret; a.gammas = gammas; a.lambdas = lambdas;
    a.done = done; a.gamma = (float)gamma; a.lambda = (float)lambda_; a.upgo_mode = upgo_mode; a.T = T; a.B = B;
    a.g_value = grad_value; a.g_reward = grad_reward; a.g_gammas = grad_gammas; a.g_lambdas = grad_lambdas;
    constexpr int NT = 64;
    return launch_k(lambda_returns_bwd_kernel<NT>, div_up(B, NT), NT, 0, (cudaStream_t)stream, a);
}

extern "C" int b200rl_td_lambda_fwd(const float* value, const float* reward, const float* weight, double gamma,
                                    double lambda_, long long T, long long B, float* loss, float* dvalue_saved,
                                    float* workspace, size_t workspace_bytes, void* stream) {
    if (T <= 0 || B <= 0 || !value || !reward || !loss || !dvalue_saved || !workspace) return B200RL_ERR_ARG;
    LamArgs a{};
    a.value = value; a.reward = reward; a.weight = weight; a.gamma = (float)gamma; a.lambda = (float)lambda_;
    a.T = T; a.B = B; a.loss = loss; a.dvalue = dvalue_saved;
    if (!ws_partials_fit((long long)(div_up(B, 8)), workspace_bytes)) return B200RL_ERR_WORKSPACE;
    return launch_lambda<0, 1>(a, workspace, (cudaStream_t)stream);
}

// COMA's value half (HEAD 2): T, B, A, N are coma_error's (T, B, A, N); the scan covers rows t < T-1.  Launched by
// b200rl_coma_fwd (csrc/pg.cu) ahead of the policy head, which reads dq.
namespace b200rl {
int launch_coma_value(const float* q, const float* target_q, const long long* action, const float* reward,
                      const float* weight, double gamma, double lambda_, long long T, long long B, long long A, long long N,
                      float* loss, float* dq, float* dret, float* ws, size_t ws_bytes, cudaStream_t st) {
    ComaLamArgs a{};
    a.reward = reward; a.weight = weight; a.gamma = (float)gamma; a.lambda = (float)lambda_;
    a.T = T - 1; a.B = B * A; a.loss = loss;
    a.action = action; a.target_q = target_q; a.q = q; a.A = A; a.N = (int)N; a.dq = dq; a.dret = dret;
    if (a.B >= 16 * 2 * NUM_SMS) {
        if (!ws_partials_fit(div_up(a.B, 16), ws_bytes)) return B200RL_ERR_WORKSPACE;
        return launch_k(lambda_scan_coma_kernel<16, 256, 64>, div_up(a.B, 16), 256, 0, st, a, ws);
    }
    if (!ws_partials_fit(div_up(a.B, 8), ws_bytes)) return B200RL_ERR_WORKSPACE;
    return launch_k(lambda_scan_coma_kernel<8, 256, 128>, div_up(a.B, 8), 256, 0, st, a, ws);
}
}  // namespace b200rl

extern "C" int b200rl_scale(const float* g, const float* in, float* out, long long n, void* stream) {
    if (n < 0 || !g || (n > 0 && (!in || !out))) return B200RL_ERR_ARG;
    if (n == 0) return B200RL_OK;
    return launch_k(scale_kernel, div_up(n, 256), 256, 0, (cudaStream_t)stream, g, in, out, n);
}
