// ACER heads: acer_policy_error (ding/rl_utils/acer.py:8-57), acer_value_error (:60-83), acer_trust_region_update (:86-124).
// Per-transition (un-reduced) outputs, as the reference returns them -- ACERPolicy applies its own weights and sums
// (policy/acer.py:247-270).  thread = transition, grid-stride; rows of N logits are read straight from global memory (the row
// is N * 4 contiguous bytes per thread; launch-bound at ACER's batch sizes).
//
//   actor_loss[tb] = min(ratio[tb, a], c) * (Qret[tb] - V[tb]) * logpi[tb, a]
//   bias_loss[tb]  = sum_j max(1 - c / (ratio[tb, j] + 1e-8), 0) * exp(logpi[tb, j]).detach() * (Q[tb, j] - V[tb]) * logpi[tb, j]
//   critic_loss[tb] = 0.5 * (Qret[tb] - Q[tb, a])^2
// Gradients flow to logpi (`target_logit`) and to Q (`q_values`, critic loss only): everything else is computed under
// torch.no_grad() or is data in the reference.
#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {

constexpr float ACER_EPS = 1e-8f;

// torch.clamp keeps NaN; fminf / fmaxf would return the other operand
__device__ __forceinline__ float clamp_max_nan(float x, float hi) { return x != x ? x : fminf(x, hi); }
__device__ __forceinline__ float clamp_min_nan(float x, float lo) { return x != x ? x : fmaxf(x, lo); }

__global__ void __launch_bounds__(256) acer_policy_fwd_kernel(const float* __restrict__ q, const float* __restrict__ qret,
                                                              const float* __restrict__ v, const float* __restrict__ logit,
                                                              const long long* __restrict__ act,
                                                              const float* __restrict__ ratio, long long M, int N, float c,
                                                              float* __restrict__ actor, float* __restrict__ bias) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const long long a = act[i];
        const float vv = v[i];
        const float* lg = logit + i * N;
        const float* rt = ratio + i * N;
        const float* qq = q + i * N;
        actor[i] = fmul(fmul(clamp_max_nan(rt[a], c), fsub(qret[i], vv)), lg[a]);
        float s = 0.f;
        for (int j = 0; j < N; ++j) {
            const float w = clamp_min_nan(fsub(1.0f, __fdiv_rn(c, fadd(rt[j], ACER_EPS))), 0.f);
            s = fadd(s, fmul(fmul(fmul(w, expf(lg[j])), fsub(qq[j], vv)), lg[j]));
        }
        bias[i] = s;
    }
}

// d (g_actor . actor + g_bias . bias) / d logpi; exp(logpi) is detached in the bias term (acer.py:52)
__global__ void __launch_bounds__(256) acer_policy_bwd_kernel(const float* __restrict__ q, const float* __restrict__ qret,
                                                              const float* __restrict__ v, const float* __restrict__ logit,
                                                              const long long* __restrict__ act,
                                                              const float* __restrict__ ratio, const float* __restrict__ g_actor,
                                                              const float* __restrict__ g_bias, long long M, int N, float c,
                                                              float* __restrict__ grad_logit) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const long long a = act[i];
        const float vv = v[i];
        const float ga = g_actor ? g_actor[i] : 0.f, gb = g_bias ? g_bias[i] : 0.f;
        const float* lg = logit + i * N;
        const float* rt = ratio + i * N;
        const float* qq = q + i * N;
        float* go = grad_logit + i * N;
        // a loss with no upstream gradient is not in the graph: it contributes nothing, not 0 * (a non-finite term)
        const float ca = g_actor ? ga * (clamp_max_nan(rt[a], c) * (qret[i] - vv)) : 0.f;
        for (int j = 0; j < N; ++j) {
            const float w = clamp_min_nan(1.0f - c / (rt[j] + ACER_EPS), 0.f);
            float g = g_bias ? gb * (w * expf(lg[j]) * (qq[j] - vv)) : 0.f;
            if (j == a && g_actor) g += ca;
            go[j] = g;
        }
    }
}

__global__ void __launch_bounds__(256) acer_value_fwd_kernel(const float* __restrict__ q, const float* __restrict__ qret,
                                                             const long long* __restrict__ act, long long M, int N,
                                                             float* __restrict__ loss) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const float d = fsub(qret[i], q[i * N + act[i]]);
        loss[i] = fmul(0.5f, fmul(d, d));
    }
}

__global__ void __launch_bounds__(256) acer_value_bwd_kernel(const float* __restrict__ q, const float* __restrict__ qret,
                                                             const long long* __restrict__ act, const float* __restrict__ g,
                                                             long long M, int N, float* __restrict__ grad_q) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const long long a = act[i];
        const float d = qret[i] - q[i * N + a];
        float* go = grad_q + i * N;
        for (int j = 0; j < N; ++j) go[j] = (j == a) ? -d * g[i] : 0.f;
    }
}

// scale = max(((g . k) - delta) / (k . k), 0),  out = g - scale * k,  k = exp(avg_logit)   (acer.py:113-123)
__global__ void __launch_bounds__(256) acer_trust_region_kernel(const float* __restrict__ grad, const float* __restrict__ avg_logit,
                                                                long long M, int N, float delta, float* __restrict__ out) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const float* g = grad + i * N;
        const float* al = avg_logit + i * N;
        float gk = 0.f, kk = 0.f;
        for (int j = 0; j < N; ++j) {
            const float k = expf(al[j]);
            gk = fadd(gk, fmul(g[j], k));
            kk = fadd(kk, fmul(k, k));
        }
        const float scale = clamp_min_nan(__fdiv_rn(fsub(gk, delta), kk), 0.f);
        for (int j = 0; j < N; ++j) out[i * N + j] = fsub(g[j], fmul(scale, expf(al[j])));
    }
}

static int acer_grid(long long M) {
    long long g = (M + 255) / 256;
    if (g > NUM_SMS * 8) g = NUM_SMS * 8;
    return (int)(g < 1 ? 1 : g);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_acer_policy_fwd(const float* q_values, const float* q_retraces, const float* v_pred,
                                      const float* target_logit, const long long* actions, const float* ratio, long long M,
                                      long long N, double c_clip_ratio, float* actor_loss, float* bias_correction_loss,
                                      void* stream) {
    if (!q_values || !q_retraces || !v_pred || !target_logit || !actions || !ratio || !actor_loss || !bias_correction_loss ||
        M < 1 || N < 1)
        return B200RL_ERR_ARG;
    return launch_k(acer_policy_fwd_kernel, acer_grid(M), 256, 0, (cudaStream_t)stream, q_values, q_retraces, v_pred,
                    target_logit, actions, ratio, M, (int)N, (float)c_clip_ratio, actor_loss, bias_correction_loss);
}

extern "C" int b200rl_acer_policy_bwd(const float* q_values, const float* q_retraces, const float* v_pred,
                                      const float* target_logit, const long long* actions, const float* ratio,
                                      const float* g_actor, const float* g_bias, long long M, long long N,
                                      double c_clip_ratio, float* grad_target_logit, void* stream) {
    if (!q_values || !q_retraces || !v_pred || !target_logit || !actions || !ratio || !grad_target_logit || M < 1 || N < 1)
        return B200RL_ERR_ARG;
    return launch_k(acer_policy_bwd_kernel, acer_grid(M), 256, 0, (cudaStream_t)stream, q_values, q_retraces, v_pred,
                    target_logit, actions, ratio, g_actor, g_bias, M, (int)N, (float)c_clip_ratio, grad_target_logit);
}

extern "C" int b200rl_acer_value_fwd(const float* q_values, const float* q_retraces, const long long* actions, long long M,
                                     long long N, float* critic_loss, void* stream) {
    if (!q_values || !q_retraces || !actions || !critic_loss || M < 1 || N < 1) return B200RL_ERR_ARG;
    return launch_k(acer_value_fwd_kernel, acer_grid(M), 256, 0, (cudaStream_t)stream, q_values, q_retraces, actions, M, (int)N,
                    critic_loss);
}

extern "C" int b200rl_acer_value_bwd(const float* q_values, const float* q_retraces, const long long* actions,
                                     const float* g_loss, long long M, long long N, float* grad_q_values, void* stream) {
    if (!q_values || !q_retraces || !actions || !g_loss || !grad_q_values || M < 1 || N < 1) return B200RL_ERR_ARG;
    return launch_k(acer_value_bwd_kernel, acer_grid(M), 256, 0, (cudaStream_t)stream, q_values, q_retraces, actions, g_loss, M,
                    (int)N, grad_q_values);
}

extern "C" int b200rl_acer_trust_region(const float* actor_gradient, const float* avg_logit, long long M, long long N,
                                        double trust_region_value, float* out, void* stream) {
    if (!actor_gradient || !avg_logit || !out || M < 1 || N < 1) return B200RL_ERR_ARG;
    return launch_k(acer_trust_region_kernel, acer_grid(M), 256, 0, (cudaStream_t)stream, actor_gradient, avg_logit, M, (int)N,
                    (float)trust_region_value, out);
}
