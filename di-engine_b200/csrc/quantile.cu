// Quantile-regression n-step TD heads: qrdqn_nstep_td_error (ding/rl_utils/td.py:1098-1166), iqn_nstep_td_error (:1253-1346),
// fqf_nstep_td_error (:1359-1436).  One kernel for the three: they differ in the memory layout of the quantile tensors
// (strides), in the Huber threshold / indicator / divisor and in which axis is summed and which averaged.  FQF's other loss,
// the fraction loss (fqf_calculate_fraction_loss, :1466-1513), has its own kernel at the end of the file.
//
//   theta_i   = q[b, i, action_b]                         i < n_i   (current quantiles, differentiable)
//   theta'_j  = R_b + g_b * next_n_q[b, j, next_action_b] * (1 - done_b)      j < n_j   (n-step target, td.py:1150-1159)
//   u_ij      = theta'_j - theta_i
//   rho_ij    = |tau_i - 1[u_ij <= 0 | < 0]| * huber_kappa(u_ij) / divisor
//   loss_b    = norm * sum_ij rho_ij     (norm = 1/n_i for QR-DQN: sum over j, mean over i; 1/n_j for IQN / FQF)
//   loss      = mean_b(loss_b * weight_b)
//
// Replay-buffer batch sizes (B = 32..512, 8..200 quantiles): launch / latency bound.  A CTA takes one sample at a time
// (grid-stride), theta / theta' / tau live in shared memory, thread = i runs over j; ONE launch writes the loss, the per-sample
// losses, d loss_b / d theta_i (for the backward pass) and, for a unit upstream gradient, the full gradient tensor
// (zeros off the chosen action) -- the backward launch verifies the upstream gradient on the device and exits.
#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {

constexpr int QT_NT = 128;

struct QtdArgs {
    const float* q;
    const float* nq;
    const long long* act;
    const long long* nact;
    const float* reward;  // (nstep, B)
    const float* done;    // (B)
    const float* tau;     // strided (b, i)
    const float* weight;  // nullable (B)
    const float* vgamma;  // nullable, stride vg_stride (0 = one value for the batch)
    long long B, N;
    int ni, nj, nstep;
    long long q_sb, q_si, q_sa, nq_sb, nq_sj, nq_sa, tau_sb, tau_si, vg_stride;
    float gamma, gamma_n, kappa, divisor, norm;
    int strict;  // indicator u < 0 (IQN, FQF) instead of u <= 0 (QR-DQN)
    float* loss;
    float* td;         // (B)
    float* dtheta;     // (B, ni)  d loss_b / d theta_i
    float* grad_unit;  // nullable, q's layout: gradient for d total / d loss = 1
};

__global__ void __launch_bounds__(QT_NT) quantile_td_kernel(QtdArgs a, float* ws) {
    pdl_prologue();
    extern __shared__ float sm[];
    float* th = sm;            // [ni]
    float* tp = th + a.ni;     // [nj]
    float* ta = tp + a.nj;     // [ni]
    __shared__ double s_red[QT_NT / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    float acc[1] = {0.f};
    const float inv_b = 1.f / (float)a.B;
    for (long long b = blockIdx.x; b < a.B; b += gridDim.x) {
        const long long ac = a.act[b], na = a.nact[b];
        // n-step return: reward_factor[k] = gamma * reward_factor[k-1] in fp32, dot product with reward[:, b] (td.py:1144-1149)
        float rf = 1.f, R = 0.f;
        for (int k = 0; k < a.nstep; ++k) {
            R = fmaf(rf, a.reward[(long long)k * a.B + b], R);
            rf = fmul(a.gamma, rf);
        }
        const float gb = a.vgamma ? a.vgamma[b * a.vg_stride] : a.gamma_n;
        const float nd = fsub(1.f, a.done[b]);
        for (int i = tid; i < a.ni; i += QT_NT) {
            th[i] = a.q[b * a.q_sb + i * a.q_si + ac * a.q_sa];
            ta[i] = a.tau[b * a.tau_sb + i * a.tau_si];
        }
        for (int j = tid; j < a.nj; j += QT_NT)
            tp[j] = fadd(R, fmul(fmul(gb, a.nq[b * a.nq_sb + j * a.nq_sj + na * a.nq_sa]), nd));
        __syncthreads();
        // the n' terms of theta_i are summed in fp64: an fp32 chain grows an error like sqrt(n') (n' up to 2048), and the
        // gradient sum cancels (d huber / d u changes sign across the target quantiles); the terms themselves stay fp32
        double lsum = 0.0;
        for (int i = tid; i < a.ni; i += QT_NT) {
            const float t = th[i], tq = ta[i];
            double li = 0.0, gi = 0.0;
            for (int j = 0; j < a.nj; ++j) {
                const float u = tp[j] - t;
                const float au = fabsf(u);
                const bool quad = a.strict == 1 ? (au <= a.kappa) : (au < a.kappa);  // torch.where(<=) vs smooth_l1 (<)
                const float hub = quad ? 0.5f * u * u : a.kappa * (au - 0.5f * a.kappa);
                const float dh = quad ? u : (u > 0.f ? a.kappa : -a.kappa);  // d huber / d u
                const bool ind = a.strict ? (u < 0.f) : (u <= 0.f);
                const float w = fabsf(tq - (ind ? 1.f : 0.f));
                li = fma((double)w, (double)hub, li);
                gi = fma((double)w, (double)dh, gi);
            }
            lsum += li;
            const float dti = (float)(-gi * (double)a.norm / (double)a.divisor);  // d u / d theta_i = -1
            a.dtheta[b * a.ni + i] = dti;
            th[i] = dti;  // own slot: the gradient pass below reads it back
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if (lane == 0) s_red[wid] = lsum;
        __syncthreads();
        double tot = 0.0;
#pragma unroll
        for (int w = 0; w < QT_NT / 32; ++w) tot += s_red[w];
        const float lb = (float)(tot * (double)a.norm / (double)a.divisor);
        const float wb = a.weight ? a.weight[b] : 1.f;
        if (tid == 0) {
            a.td[b] = lb;
            acc[0] += lb * wb;
        }
        if (a.grad_unit) {
            const float c = wb * inv_b;
            const long long n = (long long)a.ni * a.N;
            if (a.q_sa == 1) {
                for (long long e = tid; e < n; e += QT_NT) {
                    const long long i = e / a.N, x = e - i * a.N;
                    a.grad_unit[b * a.q_sb + i * a.q_si + x] = (x == ac) ? c * th[i] : 0.f;
                }
            } else {
                for (long long e = tid; e < n; e += QT_NT) {
                    const long long x = e / a.ni, i = e - x * a.ni;
                    a.grad_unit[b * a.q_sb + i * a.q_si + x * a.q_sa] = (x == ac) ? c * th[i] : 0.f;
                }
            }
        }
        __syncthreads();
    }
    float* loss = a.loss;
    grid_sum_fx<1, QT_NT>(acc, ws, [=](int, double tot) { *loss = (float)(tot * (double)inv_b); });
}

struct QtdBwdArgs {
    const float* dtheta;
    const float* weight;
    const long long* act;
    const float* g_loss;  // nullable = 0
    const float* g_td;    // nullable (B)
    long long B, N;
    int ni;
    long long q_sb, q_si, q_sa;
    int skip_if_unit;
    float* grad_q;
};

__global__ void __launch_bounds__(256) quantile_td_bwd_kernel(QtdBwdArgs a) {
    pdl_prologue();
    const float gl = a.g_loss ? *a.g_loss : 0.f;
    if (a.skip_if_unit && gl == 1.f) return;  // the forward launch already wrote exactly this gradient
    const float inv_b = 1.f / (float)a.B;
    const long long per = (long long)a.ni * a.N, n = a.B * per;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const long long b = e / per, r = e - b * per;
        long long i, x;
        if (a.q_sa == 1) { i = r / a.N; x = r - i * a.N; } else { x = r / a.ni; i = r - x * a.ni; }
        float g = 0.f;
        if (x == a.act[b]) {
            const float wb = a.weight ? a.weight[b] : 1.f;
            const float c = gl * wb * inv_b + (a.g_td ? a.g_td[b] : 0.f);
            g = c * a.dtheta[b * a.ni + i];
        }
        a.grad_q[b * a.q_sb + i * a.q_si + x * a.q_sa] = g;
    }
}

// FQF's fraction loss, fqf_calculate_fraction_loss (ding/rl_utils/td.py:1466-1513).  With s_i = q_tau_i[b, i, a_b] (i < N-1)
// and h_k = q_value[b, k, a_b] (k < N), both taken without gradient:
//   g_i  = where(s_i > (i == 0 ? h_0 : s_{i-1}), s_i - h_i, -(s_i - h_i))
//        + where(s_i < (i == N-2 ? h_{N-1} : s_{i+1}), s_i - h_{i+1}, -(s_i - h_{i+1}))      (strict; NaN picks the negation)
//   loss = mean_b sum_i g_i * quantiles[b, i+1]
// so d loss / d quantiles[b, i+1] = (u / B) * g_i and the end columns 0 and N get zero.  CTA x owns samples [x*NT, x*NT + NT)
// (launch_td_rows); its threads stride over their (sample, column of quantiles) pairs, so the saved g (B, N-1) and the unit
// gradient (B, N+1) are stored coalesced whatever N is, and the gathered columns are read through element strides.
struct FqfFracArgs {
    const float* qt;  // q_tau_i, strided (b, i, a)
    const float* qv;  // q_value, strided (b, k, a)
    const float* qn;  // quantiles, strided (b, k)
    const long long* act;
    long long B, A_t, A_v;  // an action outside [0, A) reads NaN
    int N;
    long long qt_sb, qt_si, qt_sa, qv_sb, qv_si, qv_sa, qn_sb, qn_si;
    float* loss;
    float* g;          // (B, N-1)
    float* grad_unit;  // nullable (B, N+1): d loss / d quantiles for a unit upstream gradient
};

template <int NT>
__global__ void __launch_bounds__(NT) fqf_fraction_kernel(FqfFracArgs a, float* ws) {
    pdl_prologue();
    const float* __restrict__ qt = a.qt;
    const float* __restrict__ qv = a.qv;
    const float* __restrict__ qn = a.qn;
    float* __restrict__ g = a.g;
    float* __restrict__ gu = a.grad_unit;
    const long long r0 = (long long)blockIdx.x * NT;
    const int rows = (int)((a.B - r0) < NT ? (a.B - r0) : NT);
    const int N = a.N, W = N + 1;
    // torch's mean backward on CUDA multiplies by the fp32 reciprocal of B, then MulBackward by g
    const float inv_b = 1.f / (float)a.B;
    const float qnan = __int_as_float(0x7fffffff);
    float acc[1] = {0.f};
#pragma unroll 4
    for (int e = threadIdx.x; e < rows * W; e += NT) {
        const int r = e / W, c = e - r * W;
        const long long b = r0 + r;
        float gr = 0.f;
        if (c > 0 && c < N) {
            const int i = c - 1;
            const long long ac = a.act[b];
            const bool in_t = ac >= 0 && ac < a.A_t, in_v = ac >= 0 && ac < a.A_v;
            const float* st = qt + b * a.qt_sb + ac * a.qt_sa;
            const float* hv = qv + b * a.qv_sb + ac * a.qv_sa;
            const float s = in_t ? st[i * a.qt_si] : qnan;
            const float h0 = in_v ? hv[i * a.qv_si] : qnan;
            const float h1 = in_v ? hv[(i + 1) * a.qv_si] : qnan;
            const float lo = i == 0 ? h0 : (in_t ? st[(i - 1) * a.qt_si] : qnan);
            const float hi = i == N - 2 ? h1 : (in_t ? st[(i + 1) * a.qt_si] : qnan);
            const float v1 = fsub(s, h0), v2 = fsub(s, h1);
            const float gi = fadd(s > lo ? v1 : -v1, s < hi ? v2 : -v2);
            g[b * (N - 1) + i] = gi;
            acc[0] += fmul(gi, qn[b * a.qn_sb + c * a.qn_si]);
            gr = fmul(inv_b, gi);
        }
        if (gu) gu[b * W + c] = gr;
    }
    float* loss = a.loss;
    const double nb = (double)a.B;
    td_loss_sum<1, NT>(acc, ws, false, [=](int, double tot) { *loss = (float)(tot / nb); });
}

struct FqfFracBwdArgs {
    const float* g;       // (B, N-1), saved by the forward launch
    const float* g_loss;  // device scalar
    long long B;
    int N, skip_if_unit;
    float* grad;  // (B, N+1)
};

__global__ void __launch_bounds__(256) fqf_fraction_bwd_kernel(FqfFracBwdArgs a) {
    pdl_prologue();
    const float u = *a.g_loss;
    if (a.skip_if_unit && u == 1.f) return;  // the forward launch already wrote exactly this gradient
    const float c = fmul(u, 1.f / (float)a.B);  // (u / B) as torch's mean backward forms it on CUDA, then times g
    const long long W = a.N + 1, n = a.B * W;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const long long b = e / W, k = e - b * W;
        a.grad[e] = (k > 0 && k < a.N) ? fmul(c, a.g[b * (a.N - 1) + k - 1]) : 0.f;
    }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_quantile_td_fwd(const float* q, const float* next_n_q, const long long* action,
                                      const long long* next_n_action, const float* reward, const float* done,
                                      const float* tau, const float* weight, const float* value_gamma,
                                      long long vg_stride, long long B, long long N, long long n_tau,
                                      long long n_tau_prime, long long nstep, double gamma, long long q_sb, long long q_si,
                                      long long q_sa, long long nq_sb, long long nq_sj, long long nq_sa, long long tau_sb,
                                      long long tau_si, int form, double kappa, float* loss, float* td, float* dtheta,
                                      float* grad_q_unit, float* workspace, size_t workspace_bytes, void* stream) {
    if (!q || !next_n_q || !action || !next_n_action || !reward || !done || !tau || !loss || !td || !dtheta || !workspace)
        return B200RL_ERR_ARG;
    if (B < 1 || N < 1 || n_tau < 1 || n_tau_prime < 1 || nstep < 1 || form < 0 || form > 2 || !(kappa > 0.0))
        return B200RL_ERR_ARG;
    if (n_tau > 2048 || n_tau_prime > 2048) return B200RL_ERR_ARG;  // shared-memory budget of one CTA (default 48 KB)
    if (workspace_bytes < WS_MIN_BYTES) return B200RL_ERR_WORKSPACE;
    QtdArgs a{};
    a.q = q; a.nq = next_n_q; a.act = action; a.nact = next_n_action; a.reward = reward; a.done = done; a.tau = tau;
    a.weight = weight; a.vgamma = value_gamma; a.vg_stride = vg_stride; a.B = B; a.N = N; a.ni = (int)n_tau;
    a.nj = (int)n_tau_prime; a.nstep = (int)nstep; a.q_sb = q_sb; a.q_si = q_si; a.q_sa = q_sa; a.nq_sb = nq_sb;
    a.nq_sj = nq_sj; a.nq_sa = nq_sa; a.tau_sb = tau_sb; a.tau_si = tau_si;
    a.gamma = (float)gamma;
    double gn = 1.0;
    for (long long k = 0; k < nstep; ++k) gn *= gamma;  // python: gamma ** nstep in double (td.py:1152)
    a.gamma_n = (float)gn;
    // form 0 = QR-DQN: smooth_l1 (beta 1), indicator u <= 0, sum over j / mean over i (td.py:1162-1164)
    // form 1 = IQN: huber kappa via torch.where(|u| <= kappa), indicator u < 0, / kappa, sum over i / mean over j (:1328-1344)
    // form 2 = FQF: smooth_l1 (beta 1), indicator u < 0, / kappa, sum over i / mean over j (:1422-1434)
    a.kappa = form == 1 ? (float)kappa : 1.f;
    a.divisor = form == 0 ? 1.f : (float)kappa;
    a.norm = 1.f / (float)(form == 0 ? n_tau : n_tau_prime);
    a.strict = form == 0 ? 0 : (form == 1 ? 1 : 2);
    a.loss = loss; a.td = td; a.dtheta = dtheta; a.grad_unit = grad_q_unit;
    const int grid = (int)(B < (long long)FX_MAX_GRID ? B : (long long)FX_MAX_GRID);
    const size_t smem = (size_t)(2 * n_tau + n_tau_prime) * sizeof(float);
    return launch_k(quantile_td_kernel, grid, QT_NT, smem, (cudaStream_t)stream, a, workspace);
}

extern "C" int b200rl_quantile_td_bwd(const float* dtheta, const float* weight, const long long* action, const float* g_loss,
                                      const float* g_td, long long B, long long N, long long n_tau, long long q_sb,
                                      long long q_si, long long q_sa, int skip_if_unit, float* grad_q, void* stream) {
    if (!dtheta || !action || !grad_q || B < 1 || N < 1 || n_tau < 1) return B200RL_ERR_ARG;
    QtdBwdArgs a{};
    a.dtheta = dtheta; a.weight = weight; a.act = action; a.g_loss = g_loss; a.g_td = g_td; a.B = B; a.N = N;
    a.ni = (int)n_tau; a.q_sb = q_sb; a.q_si = q_si; a.q_sa = q_sa; a.skip_if_unit = (skip_if_unit && !g_td) ? 1 : 0;
    a.grad_q = grad_q;
    const long long n = B * N * n_tau;
    long long grid = (n + 255) / 256;
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    return launch_k(quantile_td_bwd_kernel, (int)grid, 256, 0, (cudaStream_t)stream, a);
}

extern "C" int b200rl_fqf_fraction_fwd(const float* q_tau_i, const float* q_value, const float* quantiles,
                                       const long long* actions, long long B, long long N, long long A_tau,
                                       long long A_value, long long qt_sb, long long qt_si, long long qt_sa, long long qv_sb,
                                       long long qv_si, long long qv_sa, long long qn_sb, long long qn_si, float* loss,
                                       float* g_saved, float* grad_quantiles_unit, float* workspace, size_t workspace_bytes,
                                       void* stream) {
    if (!q_tau_i || !q_value || !quantiles || !actions || !loss || !g_saved || !workspace) return B200RL_ERR_ARG;
    // N <= 2^20: a CTA's (sample, column) pairs, at most 1024 * (N + 1), are counted in int
    if (B < 1 || N < 1 || N > (1 << 20) || A_tau < 1 || A_value < 1) return B200RL_ERR_ARG;
    FqfFracArgs a{};
    a.qt = q_tau_i; a.qv = q_value; a.qn = quantiles; a.act = actions; a.B = B; a.A_t = A_tau; a.A_v = A_value;
    a.N = (int)N; a.qt_sb = qt_sb; a.qt_si = qt_si; a.qt_sa = qt_sa; a.qv_sb = qv_sb; a.qv_si = qv_si; a.qv_sa = qv_sa;
    a.qn_sb = qn_sb; a.qn_si = qn_si; a.loss = loss; a.g = g_saved; a.grad_unit = grad_quantiles_unit;
    return launch_td_rows<1>([](auto nt) { return fqf_fraction_kernel<decltype(nt)::value>; }, a, B, false, workspace,
                             workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200rl_fqf_fraction_bwd(const float* g_saved, const float* g_loss, long long B, long long N,
                                       int skip_if_unit, float* grad_quantiles, void* stream) {
    if (!g_saved || !g_loss || !grad_quantiles || B < 1 || N < 1) return B200RL_ERR_ARG;
    FqfFracBwdArgs a{};
    a.g = g_saved; a.g_loss = g_loss; a.B = B; a.N = (int)N; a.skip_if_unit = skip_if_unit ? 1 : 0;
    a.grad = grad_quantiles;
    const long long n = B * (N + 1);
    long long grid = (n + 255) / 256;
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    return launch_k(fqf_fraction_bwd_kernel, (int)grid, 256, 0, (cudaStream_t)stream, a);
}
