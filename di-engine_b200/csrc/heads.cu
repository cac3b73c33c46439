// Sibling loss heads of the hot path (SURVEY section 8f rank 3), each forward + gradients in ONE launch:
//   a2c_error              ding/rl_utils/a2c.py:10-44      policy -mean(logp*adv*w), value mean(w*(ret-v)^2), entropy mean(H*w)
//   a2c_error_continuous   ding/rl_utils/a2c.py:50-88      the same three losses on an Independent(Normal(mu, sigma)) policy
//   ppo_error_continuous   ding/rl_utils/ppo.py:278-374    the PPO loss of ppo.cu on an Independent(Normal(mu, sigma)) policy
// Scheme of the other heads: thread = row, grid-stride, the forward launch also writes the gradients for the upstream
// gradients it expects (the loss weights of the training loop, remembered on the device); the backward launch is the same
// kernel in verify mode -- it returns at once when the actual upstream gradients are the recorded ones and recomputes
// otherwise (exact for any upstream gradient, no host sync).  Loss sums: one atomic round trip per CTA (grid_sum_fx).
#include <math.h>

#include "../../include/b200rl.h"
#include "ppo_math.cuh"

namespace b200rl {

constexpr int HD_NT = 256;
constexpr float kLogSqrt2Pi = 0.9189385332046727f;       // math.log(math.sqrt(2 * math.pi))
constexpr float kHalfPlusHalfLog2Pi = 1.4189385332046727f;  // 0.5 + 0.5 * math.log(2 * math.pi)

// ---------------------------------------------------------------------------------------------------------------
// a2c_error (discrete)
// ---------------------------------------------------------------------------------------------------------------
struct A2cArgs {
    const float* logit;       // (S, N)
    const long long* action;  // (S)
    const float* value;       // (S)
    const float* adv;         // (S)
    const float* ret;         // (S)
    const float* weight;      // nullable (S)
    long long S;
    int N;
    float* out;         // 3 losses
    float* grad_logit;  // nullable: losses only
    float* grad_value;
    UpstreamRecord rec;  // slots policy, value, entropy
};

__global__ void __launch_bounds__(HD_NT) a2c_kernel(A2cArgs a, float* ws) {
    pdl_prologue();
    float g[3];
    if (upstream<3>(a.rec, a.rec.verify, 7u, g)) return;
    const bool grads = a.grad_logit != nullptr;
    const float inv_s = 1.f / (float)a.S;
    float acc[3] = {0.f, 0.f, 0.f};
    for (long long s = (long long)blockIdx.x * HD_NT + threadIdx.x; s < a.S; s += (long long)gridDim.x * HD_NT) {
        const float* z = a.logit + s * a.N;
        const int act = (int)a.action[s];
        const float w = a.weight ? a.weight[s] : 1.f;
        const float adv = a.adv[s], v = a.value[s], ret = a.ret[s];
        float lse, ent;
        row_lse_entropy<1>([&](int j) { return z[j]; }, a.N, 0, lse, ent);
        const float lp = z[act] - lse;
        const float dv = ret - v;
        acc[0] -= lp * adv * w;
        acc[1] += dv * dv * w;
        acc[2] += ent * w;
        if (grads) {
            const float c_act = g[0] * (-adv * w) * inv_s, c_ent = g[2] * w * inv_s;
            float* gz = a.grad_logit + s * a.N;
            for (int j = 0; j < a.N; ++j) {
                const float lpj = fmaxf(z[j] - lse, kF32Min);  // Categorical.entropy's clamp: 0 * finite at a -inf logit
                const float p = expf(lpj);
                float gj = -c_act * p - c_ent * p * (lpj + ent);
                if (j == act) gj += c_act;
                gz[j] = gj;
            }
            a.grad_value[s] = g[1] * (-2.f * w * dv) * inv_s;
        }
    }
    if (a.rec.verify) return;  // the losses were written by the forward launch
    const double is = 1.0 / (double)a.S;
    grid_sum_fx<3, HD_NT>(acc, ws, [&](int k, double t) { a.out[k] = (float)(t * is); });
}

// ---------------------------------------------------------------------------------------------------------------
// ppo_error_continuous
// ---------------------------------------------------------------------------------------------------------------
struct PpocArgs {
    const float* mu_new;     // (S, D)
    const float* sigma_new;  // (S, D)
    const float* mu_old;     // (S, D)
    const float* sigma_old;
    const float* mu_pre;     // nullable (S, D)
    const float* sigma_pre;
    const float* action;     // (S, D)
    const float* value_new;  // (S)
    const float* value_old;
    const float* adv;
    const float* ret;
    const float* weight;  // nullable
    // nullable (S): happo_error_continuous (ding/rl_utils/happo.py:195-284): min(surr1, surr2) * factor before the dual clip,
    // and the entropy / approx_kl means run over the S * D per-dimension terms (Normal instead of Independent(Normal))
    const float* factor;
    long long S;
    int D;
    float clip, clip_lo, clip_hi, dual_clip;
    int use_value_clip, kl_type;
    float* out;  // 6: policy, value, entropy, kl, approx_kl, clipfrac
    float* grad_mu;     // nullable: losses only
    float* grad_sigma;
    float* grad_value;
    UpstreamRecord rec;  // slots policy, value, entropy, and kl with the pretrained policy
};

// log N(a; mu, sigma) summed over the D action dims, torch.distributions.Normal.log_prob's expression
__device__ __forceinline__ float normal_logp(const float* mu, const float* sg, const float* ac, int D) {
    float lp = 0.f;
    for (int d = 0; d < D; ++d) {
        const float df = ac[d] - mu[d], s = sg[d];
        lp += -(df * df) / (2.f * s * s) - logf(s) - kLogSqrt2Pi;
    }
    return lp;
}

__global__ void __launch_bounds__(HD_NT) ppoc_kernel(PpocArgs a, float* ws) {
    pdl_prologue();
    float g[4];
    const bool grads = a.grad_mu != nullptr, has_pre = a.mu_pre != nullptr;
    if (upstream<4>(a.rec, a.rec.verify, has_pre ? 15u : 7u, g)) return;
    const float inv_s = 1.f / (float)a.S;
    const float ent_scale = a.factor ? 1.f / (float)a.D : 1.f;  // happo: mean over S * D elements
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long s = (long long)blockIdx.x * HD_NT + threadIdx.x; s < a.S; s += (long long)gridDim.x * HD_NT) {
        const long long o = s * a.D;
        const float* mu = a.mu_new + o;
        const float* sg = a.sigma_new + o;
        const float* ac = a.action + o;
        const float w = a.weight ? a.weight[s] : 1.f;
        const float lp_n = normal_logp(mu, sg, ac, a.D);
        const float lp_o = normal_logp(a.mu_old + o, a.sigma_old + o, ac, a.D);
        float ent = 0.f;
        for (int d = 0; d < a.D; ++d) ent += kHalfPlusHalfLog2Pi + logf(sg[d]);
        const float ratio = expf(lp_n - lp_o);
        float dsel, dterm, dk = 0.f, klv = 0.f;
        const float sel = surrogate(ratio, a.adv[s], a.clip_lo, a.clip_hi, a.dual_clip, dsel, true, a.factor ? a.factor[s] : 1.f);
        const float vt = value_term(a.value_new[s], a.value_old[s], a.ret[s], a.clip, a.use_value_clip, dterm);
        if (has_pre) klv = kl_term(lp_n - normal_logp(a.mu_pre + o, a.sigma_pre + o, ac, a.D), a.kl_type, dk);
        acc[0] -= sel * w;
        acc[1] += vt * w;
        acc[2] += ent * w;
        acc[3] += klv;
        acc[4] += lp_o - lp_n;
        acc[5] += (ratio > a.clip_hi || ratio < a.clip_lo) ? 1.f : 0.f;
        if (grads) {
            const float c_lp = g[0] * (-w * inv_s) * dsel * ratio + g[3] * dk * inv_s;  // d total / d logp_new
            const float c_ent = g[2] * w * inv_s * ent_scale;                             // d total / d entropy
            for (int d = 0; d < a.D; ++d) {
                const float sd = sg[d], df = ac[d] - mu[d], inv = 1.f / sd;
                a.grad_mu[o + d] = c_lp * df * inv * inv;
                a.grad_sigma[o + d] = c_lp * (df * df * inv * inv * inv - inv) + c_ent * inv;
            }
            a.grad_value[s] = g[1] * 0.5f * w * inv_s * dterm;
        }
    }
    if (a.rec.verify) return;
    const double is = 1.0 / (double)a.S;
    const double per_dim = a.factor ? 1.0 / (double)a.D : 1.0;
    grid_sum_fx<6, HD_NT>(acc, ws, [&](int k, double t) {
        double sc = k == 1 ? 0.5 * is : (k == 3 && !has_pre ? 0.0 : is);
        if (k == 2 || k == 4) sc *= per_dim;
        a.out[k] = (float)(t * sc);
    });
}

// ---------------------------------------------------------------------------------------------------------------
// a2c_error_continuous: a2c_kernel's three losses on an Independent(Normal(mu, sigma)) policy
// ---------------------------------------------------------------------------------------------------------------
struct A2ccArgs {
    const float* mu;      // (S, D)
    const float* sigma;   // (S, D)
    const float* action;  // (S, D)
    const float* value;   // (S)
    const float* adv;     // (S)
    const float* ret;     // (S)
    const float* weight;  // nullable (S)
    long long S;
    int D;
    float* out;        // 3 losses
    float* grad_mu;    // nullable: losses only
    float* grad_sigma;
    float* grad_value;
    UpstreamRecord rec;  // slots policy, value, entropy
};

__global__ void __launch_bounds__(HD_NT) a2cc_kernel(A2ccArgs a, float* ws) {
    pdl_prologue();
    float g[3];
    if (upstream<3>(a.rec, a.rec.verify, 7u, g)) return;
    const bool grads = a.grad_mu != nullptr;
    const float inv_s = 1.f / (float)a.S;
    float acc[3] = {0.f, 0.f, 0.f};
    for (long long s = (long long)blockIdx.x * HD_NT + threadIdx.x; s < a.S; s += (long long)gridDim.x * HD_NT) {
        const long long o = s * a.D;
        const float* mu = a.mu + o;
        const float* sg = a.sigma + o;
        const float* ac = a.action + o;
        const float w = a.weight ? a.weight[s] : 1.f;
        const float adv = a.adv[s], v = a.value[s], ret = a.ret[s];
        const float lp = normal_logp(mu, sg, ac, a.D);
        float ent = 0.f;
        for (int d = 0; d < a.D; ++d) ent += kHalfPlusHalfLog2Pi + logf(sg[d]);
        const float dv = ret - v;
        acc[0] -= lp * adv * w;
        acc[1] += dv * dv * w;
        acc[2] += ent * w;
        if (grads) {
            const float c_lp = g[0] * (-adv * w) * inv_s, c_ent = g[2] * w * inv_s;
            for (int d = 0; d < a.D; ++d) {
                const float sd = sg[d], df = ac[d] - mu[d], inv = 1.f / sd;
                a.grad_mu[o + d] = c_lp * df * inv * inv;
                a.grad_sigma[o + d] = c_lp * (df * df * inv * inv * inv - inv) + c_ent * inv;
            }
            a.grad_value[s] = g[1] * (-2.f * w * dv) * inv_s;
        }
    }
    if (a.rec.verify) return;
    const double is = 1.0 / (double)a.S;
    grid_sum_fx<3, HD_NT>(acc, ws, [&](int k, double t) { a.out[k] = (float)(t * is); });
}

// ---------------------------------------------------------------------------------------------------------------
// ppg_joint_error's behavioural-cloning term (ding/rl_utils/ppg.py:62-67): F.kl_div(logp_new, logp_old, 'batchmean') with the
// LOG-probability of the old policy passed as the (non-log) target, exactly as the reference does:
//   loss = (1/B) sum_b [ xlogy(t_b, t_b) - t_b * x_b ],   x_b = log pi_new(a_b), t_b = log pi_old(a_b) <= 0
// xlogy(t, t) is NaN for t < 0, so the VALUE is NaN whenever any old log-probability is negative (as in the reference); the
// GRADIENT d loss / d x_b = -t_b / B is finite and is what PPG trains on.  dlogit_unit = that gradient through log-softmax.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(HD_NT) ppg_bc_kernel(const float* __restrict__ logit_new, const float* __restrict__ logit_old,
                                                       const long long* __restrict__ action, long long B, int N,
                                                       float* __restrict__ loss, float* __restrict__ dlogit_unit, float* ws) {
    pdl_prologue();
    float acc[1] = {0.f};
    const float inv_b = 1.f / (float)B;
    for (long long b = (long long)blockIdx.x * HD_NT + threadIdx.x; b < B; b += (long long)gridDim.x * HD_NT) {
        const float* zn = logit_new + b * N;
        const float* zo = logit_old + b * N;
        const long long a = action[b];
        float mn = kF32Min, mo = kF32Min;
        for (int j = 0; j < N; ++j) { mn = fmaxf(mn, zn[j]); mo = fmaxf(mo, zo[j]); }
        float sn = 0.f, so = 0.f;
        for (int j = 0; j < N; ++j) { sn += expf(zn[j] - mn); so += expf(zo[j] - mo); }
        const float lse_n = mn + logf(sn);
        const float x = zn[a] - lse_n, t = (zo[a] - mo) - logf(so);
        acc[0] += (t == 0.f ? 0.f : t * logf(t)) - t * x;  // xlogy(t, t) - t * x
        if (dlogit_unit) {
            const float c = -t * inv_b;
            float* g = dlogit_unit + b * N;
            for (int j = 0; j < N; ++j) g[j] = c * ((j == a ? 1.f : 0.f) - expf(zn[j] - lse_n));
        }
    }
    grid_sum_fx<1, HD_NT>(acc, ws, [=](int, double tot) { *loss = (float)(tot * (double)inv_b); });
}

static int head_grid(long long S) {
    long long grid = div_up(S, HD_NT);
    if (grid > NUM_SMS * 3) grid = NUM_SMS * 3;  // <= 511 CTAs: the one-round-trip reduction applies
    return (int)(grid < 1 ? 1 : grid);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_a2c_fwd_grad(const float* logit, const long long* action, const float* value, const float* adv,
                                   const float* return_, const float* weight, long long S, long long N,
                                   const float* g_expected, int verify, const float* g_policy, const float* g_value,
                                   const float* g_entropy, float* g_used, float* g_hint, float* out3, float* grad_logit,
                                   float* grad_value, float* workspace, size_t workspace_bytes, void* stream) {
    if (S < 1 || N < 1 || !logit || !action || !value || !adv || !return_ || !workspace || workspace_bytes < WS_MIN_BYTES)
        return B200RL_ERR_ARG;
    if (!upstream_args_ok(verify, out3, grad_logit, grad_logit && grad_value, g_expected, g_used)) return B200RL_ERR_ARG;
    A2cArgs a{};
    a.logit = logit; a.action = action; a.value = value; a.adv = adv; a.ret = return_; a.weight = weight; a.S = S;
    a.N = (int)N; a.out = out3; a.grad_logit = grad_logit; a.grad_value = grad_value;
    a.rec = verify ? verify_record(g_policy, g_value, g_entropy, nullptr, g_used, g_hint)
                   : forward_record(g_expected, g_used);
    return launch_k(a2c_kernel, head_grid(S), HD_NT, 0, (cudaStream_t)stream, a, workspace);
}

extern "C" int b200rl_ppo_continuous_fwd_grad(
    const float* mu_new, const float* sigma_new, const float* mu_old, const float* sigma_old, const float* mu_pretrained,
    const float* sigma_pretrained, const float* action, const float* value_new, const float* value_old, const float* adv,
    const float* return_, const float* weight, const float* factor, long long S, long long D, double clip_ratio,
    int use_value_clip, double dual_clip, int kl_type, const float* g_expected, int verify, const float* g_policy,
    const float* g_value,
    const float* g_entropy, const float* g_kl, float* g_used, float* g_hint, float* out6, float* grad_mu, float* grad_sigma,
    float* grad_value, float* workspace, size_t workspace_bytes, void* stream) {
    if (S < 1 || D < 1 || !mu_new || !sigma_new || !mu_old || !sigma_old || !action || !value_new || !value_old || !adv ||
        !return_ || !workspace || workspace_bytes < WS_MIN_BYTES || kl_type < 1 || kl_type > 3 ||
        (!mu_pretrained) != (!sigma_pretrained))
        return B200RL_ERR_ARG;
    if (!upstream_args_ok(verify, out6, grad_mu, grad_mu && grad_sigma && grad_value, g_expected, g_used))
        return B200RL_ERR_ARG;
    PpocArgs a{};
    a.mu_new = mu_new; a.sigma_new = sigma_new; a.mu_old = mu_old; a.sigma_old = sigma_old; a.mu_pre = mu_pretrained;
    a.sigma_pre = sigma_pretrained; a.action = action; a.value_new = value_new; a.value_old = value_old; a.adv = adv;
    a.ret = return_; a.weight = weight; a.factor = factor; a.S = S; a.D = (int)D; a.clip = (float)clip_ratio;
    a.clip_lo = (float)(1.0 - clip_ratio); a.clip_hi = (float)(1.0 + clip_ratio); a.dual_clip = (float)dual_clip;
    a.use_value_clip = use_value_clip; a.kl_type = kl_type; a.out = out6; a.grad_mu = grad_mu; a.grad_sigma = grad_sigma;
    a.grad_value = grad_value;
    a.rec = verify ? verify_record(g_policy, g_value, g_entropy, g_kl, g_used, g_hint)
                   : forward_record(g_expected, g_used);
    return launch_k(ppoc_kernel, head_grid(S), HD_NT, 0, (cudaStream_t)stream, a, workspace);
}

extern "C" int b200rl_a2c_continuous_fwd_grad(const float* mu, const float* sigma, const float* action, const float* value,
                                              const float* adv, const float* return_, const float* weight, long long S,
                                              long long D, const float* g_expected, int verify, const float* g_policy,
                                              const float* g_value, const float* g_entropy, float* g_used, float* g_hint,
                                              float* out3, float* grad_mu, float* grad_sigma, float* grad_value,
                                              float* workspace, size_t workspace_bytes, void* stream) {
    if (S < 1 || D < 1 || !mu || !sigma || !action || !value || !adv || !return_ || !workspace ||
        workspace_bytes < WS_MIN_BYTES)
        return B200RL_ERR_ARG;
    if (!upstream_args_ok(verify, out3, grad_mu, grad_mu && grad_sigma && grad_value, g_expected, g_used))
        return B200RL_ERR_ARG;
    A2ccArgs a{};
    a.mu = mu; a.sigma = sigma; a.action = action; a.value = value; a.adv = adv; a.ret = return_; a.weight = weight;
    a.S = S; a.D = (int)D; a.out = out3; a.grad_mu = grad_mu; a.grad_sigma = grad_sigma; a.grad_value = grad_value;
    a.rec = verify ? verify_record(g_policy, g_value, g_entropy, nullptr, g_used, g_hint)
                   : forward_record(g_expected, g_used);
    return launch_k(a2cc_kernel, head_grid(S), HD_NT, 0, (cudaStream_t)stream, a, workspace);
}

extern "C" int b200rl_ppg_bc_fwd(const float* logit_new, const float* logit_old, const long long* action, long long B,
                                 long long N, float* loss, float* dlogit_unit, float* workspace, size_t workspace_bytes,
                                 void* stream) {
    if (B < 1 || N < 1 || !logit_new || !logit_old || !action || !loss || !workspace || workspace_bytes < WS_MIN_BYTES)
        return B200RL_ERR_ARG;
    return launch_k(ppg_bc_kernel, head_grid(B), HD_NT, 0, (cudaStream_t)stream, logit_new, logit_old, action, B, (int)N, loss,
                    dlogit_unit, workspace);
}
