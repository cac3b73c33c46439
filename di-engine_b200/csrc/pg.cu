// Policy-gradient heads on (T, B, N) logits:
//   upgo_loss (ding/rl_utils/upgo.py:77-111, tb_cross_entropy :7-43)           -> upgo_head_fwd / upgo_head_bwd
//   vtrace_error_discrete_action (ding/rl_utils/vtrace.py:72-136, isw.py:55-58) -> vtrace_fwd / vtrace_bwd
//
// V-trace forward is two launches: a row kernel (log-softmax statistics of the target and behaviour logits, one pass
// over the two (T,B,N) tensors, rows staged through shared memory) and a column-tile scan kernel (gae.cu scheme) that
// turns the importance weights into vs / advantages, reduces the three losses in-kernel and leaves the per-element
// gradient coefficients for the single backward launch.
#include "../../include/b200rl.h"
#include "ppo_math.cuh"

namespace b200rl {

// stage `nflt` contiguous floats gsrc[0..nflt) into shared memory, float4 when both sides are 16B-aligned
template <int NT>
__device__ __forceinline__ void stage_rows(float* sdst, const float* gsrc, int nflt, bool vec_ok) {
    int done = 0;
    if (vec_ok) {
        const int nv4 = nflt >> 2;
        for (int i = threadIdx.x; i < nv4; i += NT)
            reinterpret_cast<float4*>(sdst)[i] = ldg_stream4(reinterpret_cast<const float4*>(gsrc) + i);
        done = nv4 << 2;
    }
    for (int i = done + threadIdx.x; i < nflt; i += NT) sdst[i] = gsrc[i];
}

// ---------------------------------------------------------------------------------------------------------------
// UPGO head.  rows = T*B*K (K = 1 for (T,B,N) logits, K = N2 for (T,B,N2,N)); metric[t,b] = sum_k mask_k * logp(a_k);
// adv = rho * (G - V_t) with G from lambda_returns(upgo mode); loss = -mean_{T*B}(adv * metric).
// ---------------------------------------------------------------------------------------------------------------
struct UpgoArgs {
    const float* logit;       // (TB*K, N)
    const long long* action;  // (TB*K)
    const float* mask;        // nullable (TB*K)
    const float* rho;         // (TB)
    const float* ret;         // (TB) upgo returns
    const float* value;       // (TB) = bootstrap_values[:-1]
    long long TB;
    int K;
    int N;
    float* loss;
    float* adv_saved;  // (TB)
    const float* g_loss;
    float* grad_logit;
    float* grad_unit;   // forward: nullable, d loss / d logit for a unit upstream gradient (one pass over the logits)
    int skip_if_unit;   // backward: grad_logit already holds the unit gradient -> return when *g_loss == 1
};

// log softmax in torch's order, (z - max) - log(sum exp(z - max)): z - (max + log sum) loses |max| * 2^-24 on logits
// shifted far from 0 (a row shifted by 50 carried 4e-6 of error into every log-probability and probability)
template <int L, class Ld>
__device__ __forceinline__ void row_max_logsum(Ld ld, int n, int lane, float& m, float& ls) {
    m = -INFINITY;
    for (int j = lane; j < n; j += L) m = fmaxf(m, ld(j));
    if (L == 32) m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < n; j += L) s += expf(ld(j) - m);
    if (L == 32) s = warp_sum(s);
    ls = logf(s);
}

template <int NT, int L>
__global__ void __launch_bounds__(NT) upgo_fwd_kernel(UpgoArgs a, float* ws) {
    pdl_prologue();
    const int lane = (L == 32) ? (threadIdx.x & 31) : 0;
    // grid-stride over the samples: a bounded grid keeps the per-CTA loss reduction (ticket + fence) off the critical path -- one
    // CTA per four rows spent most of the kernel in it (T = B = N = 256: 16 384 CTAs)
    const long long s0 = (L == 32) ? (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5)
                                   : (long long)blockIdx.x * NT + threadIdx.x;
    const long long stride = (L == 32) ? (long long)gridDim.x * (NT / 32) : (long long)gridDim.x * NT;
    float acc[1] = {0.f};
    for (long long s = s0; s < a.TB; s += stride) {
        const float adv = fmul(a.rho[s], fsub(a.ret[s], a.value[s]));  // upgo.py:107
        float metric = 0.f;
        for (int k = 0; k < a.K; ++k) {
            const long long row = s * a.K + k;
            const float* z = a.logit + row * a.N;
            float m, ls;
            row_max_logsum<L>([&](int j) { return z[j]; }, a.N, lane, m, ls);
            const int act = (int)a.action[row];
            float lp = (z[act] - m) - ls;
            const float mk = a.mask ? a.mask[row] : 1.f;
            lp *= mk;
            metric += lp;
            if (a.grad_unit) {  // the row is still in L1: its gradient for a unit upstream gradient goes out in the same pass
                const float c = -adv * mk / (float)a.TB;  // d loss / d logp(row)
                float* gz = a.grad_unit + row * a.N;
                for (int j = lane; j < a.N; j += L) {
                    float gj = -c * expf((z[j] - m) - ls);
                    if (j == act) gj += c;
                    gz[j] = gj;
                }
            }
        }
        if (lane == 0) {
            a.adv_saved[s] = adv;
            acc[0] += adv * metric;
        }
    }
    double tot[1];
    if (grid_sum<1, NT>(acc, tot, ws, 0) && threadIdx.x == 0) a.loss[0] = (float)(-tot[0] / (double)a.TB);
}

template <int NT, int L>
__global__ void __launch_bounds__(NT) upgo_bwd_kernel(UpgoArgs a) {
    pdl_prologue();
    const int lane = (L == 32) ? (threadIdx.x & 31) : 0;
    const float g = a.g_loss ? *a.g_loss : 0.f;
    if (a.skip_if_unit && g == 1.f) return;  // the forward launch already wrote exactly this gradient
    // bounded grid-stride grid: the verification launch must be cheap (one CTA per four rows makes even an early return expensive)
    const long long r0 = (L == 32) ? (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5)
                                   : (long long)blockIdx.x * NT + threadIdx.x;
    const long long stride = (L == 32) ? (long long)gridDim.x * (NT / 32) : (long long)gridDim.x * NT;
    for (long long row = r0; row < a.TB * a.K; row += stride) {
        const long long s = row / a.K;
        const float* z = a.logit + row * a.N;
        float* gz = a.grad_logit + row * a.N;
        float m, ls;
        row_max_logsum<L>([&](int j) { return z[j]; }, a.N, lane, m, ls);
        float c = -g * a.adv_saved[s] / (float)a.TB;  // d loss / d logp(row)
        if (a.mask) c *= a.mask[row];
        const int act = (int)a.action[row];
        for (int j = lane; j < a.N; j += L) {
            float gj = -c * expf((z[j] - m) - ls);
            if (j == act) gj += c;
            gz[j] = gj;
        }
    }
}

// tb_cross_entropy (upgo.py:7-43) on its own: ce[s] = sum_k mask_k * log p(a_k) (3-D logits: K = 1, the reference's mean
// over a singleton dim) and its backward for an upstream gradient per (t, b) entry.
template <int NT, int L>
__global__ void __launch_bounds__(NT) tbce_fwd_kernel(const float* __restrict__ logit, const long long* __restrict__ action,
                                                      const float* __restrict__ mask, long long TB, int K, int N,
                                                      float* __restrict__ ce) {
    pdl_prologue();
    const int lane = (L == 32) ? (threadIdx.x & 31) : 0;
    const long long s = (L == 32) ? (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5)
                                  : (long long)blockIdx.x * NT + threadIdx.x;
    if (s >= TB) return;
    float metric = 0.f;
    for (int k = 0; k < K; ++k) {
        const long long row = s * K + k;
        const float* z = logit + row * N;
        float m, ls;
        row_max_logsum<L>([&](int j) { return z[j]; }, N, lane, m, ls);
        float lp = (z[action[row]] - m) - ls;
        if (mask) lp *= mask[row];
        metric += lp;
    }
    if (lane == 0) ce[s] = metric;
}

template <int NT, int L>
__global__ void __launch_bounds__(NT) tbce_bwd_kernel(const float* __restrict__ logit, const long long* __restrict__ action,
                                                      const float* __restrict__ mask, const float* __restrict__ g_ce,
                                                      long long TB, int K, int N, float* __restrict__ grad_logit) {
    pdl_prologue();
    const int lane = (L == 32) ? (threadIdx.x & 31) : 0;
    const long long row = (L == 32) ? (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5)
                                    : (long long)blockIdx.x * NT + threadIdx.x;
    if (row >= TB * K) return;
    const float* z = logit + row * N;
    float* gz = grad_logit + row * N;
    float m, ls;
    row_max_logsum<L>([&](int j) { return z[j]; }, N, lane, m, ls);
    float c = g_ce[row / K];
    if (mask) c *= mask[row];
    const int act = (int)action[row];
    for (int j = lane; j < N; j += L) {
        float gj = -c * expf((z[j] - m) - ls);
        if (j == act) gj += c;
        gz[j] = gj;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// V-trace
// ---------------------------------------------------------------------------------------------------------------
struct VtArgs {
    const float* target;      // (M, N) M = T*B
    const float* behaviour;   // (M, N)
    const long long* action;  // (M)
    const float* value;       // (T+1, B)
    const float* reward;      // (T, B)
    const float* weight;      // nullable (T, B)
    long long T, B;
    int N;
    float gamma, gamma_lambda, rho_clip, c_clip, rho_pg_clip;
    // forward scratch / saved (all (T, B))
    float* lp_t;     // log pi(a)
    float* isw;      // importance weight, overwritten in the scan kernel by c_pg = adv*w
    float* ent;      // row entropy, overwritten by the scan kernel with dV = 2*w*(V - vs)/M
    float* out;      // 3 losses
    // backward
    const float* g_pg;
    const float* g_val;
    const float* g_ent;
    float* grad_logit;  // (M, N)
    float* grad_value;  // (T+1, B)
};

// rows: one thread per (t,b) row; STAGED: NT consecutive rows of both logit tensors go through shared memory
template <int NT, bool STAGED>
__global__ void __launch_bounds__(NT) vtrace_rows_kernel(VtArgs a) {
    pdl_prologue();
    extern __shared__ __align__(16) float smem[];
    const int N = a.N;
    const long long M = a.T * a.B;
    const long long row0 = (long long)blockIdx.x * NT;
    const long long row = row0 + threadIdx.x;
    const float *zt, *zb;
    if (STAGED) {
        const int nflt = (int)min((long long)NT, M - row0) * N;
        stage_rows<NT>(smem, a.target + row0 * N, nflt, true);
        stage_rows<NT>(smem + NT * N, a.behaviour + row0 * N, nflt, true);
        __syncthreads();
        zt = smem + threadIdx.x * N;
        zb = smem + NT * N + threadIdx.x * N;
    } else {
        zt = a.target + row * N;
        zb = a.behaviour + row * N;
    }
    if (row >= M) return;
    const int act = (int)a.action[row];
    float lse_t, ent;
    row_lse_entropy<1>([&](int j) { return zt[j]; }, N, 0, lse_t, ent);
    const float lse_b = row_lse<1>([&](int j) { return zb[j]; }, N, 0);
    const float lp_t = zt[act] - lse_t;
    const float lp_b = zb[act] - lse_b;
    a.lp_t[row] = lp_t;
    a.isw[row] = expf(lp_t - lp_b);
    a.ent[row] = ent;
}

// large-N variant: warp per row
template <int NT>
__global__ void __launch_bounds__(NT) vtrace_rows_warp_kernel(VtArgs a) {
    pdl_prologue();
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
    if (row >= a.T * a.B) return;
    const float* zt = a.target + row * a.N;
    const float* zb = a.behaviour + row * a.N;
    const int act = (int)a.action[row];
    float lse_t, ent;
    row_lse_entropy<32>([&](int j) { return zt[j]; }, a.N, lane, lse_t, ent);
    const float lse_b = row_lse<32>([&](int j) { return zb[j]; }, a.N, lane);
    if (lane == 0) {
        const float lp_t = zt[act] - lse_t;
        a.lp_t[row] = lp_t;
        a.isw[row] = expf(lp_t - (zb[act] - lse_b));
        a.ent[row] = ent;
    }
}

// column-tile scan: x_t = delta_t + (gl*c_t)*x_{t+1}; vs_t = V_t + x_t  (vtrace.py:22-29), then
// adv_t = rho_pg*(r_t + g*vs_{t+1} - V_t) with vs_T = V_T (vtrace.py:126-128) and the three loss sums (:130-135).
// Every input of the tile is read from HBM exactly once (phase 1) and kept in shared memory for the output phase.
template <int TC, int NT, int CHUNK>
__global__ void __launch_bounds__(NT) vtrace_scan_kernel(VtArgs a, float* ws) {
    pdl_prologue();
    __shared__ float s_d[CHUNK][TC];        // delta
    __shared__ float s_f[CHUNK][TC];        // gl*c
    __shared__ float s_v[CHUNK][TC];        // V_t
    __shared__ float s_vs[CHUNK + 1][TC];   // vs_t (row `rows` = the row above the slab)
    __shared__ float s_g[CHUNK][TC];        // rho_pg, then reused for nothing else
    __shared__ float s_r[CHUNK][TC];        // reward
    __shared__ float s_w[CHUNK][TC];        // weight
    __shared__ float s_l[CHUNK][TC];        // log pi(a)
    __shared__ float s_e[CHUNK][TC];        // entropy
    const long long c0 = (long long)blockIdx.x * TC;
    const long long T = a.T, B = a.B;
    const float inv_m = 1.f / (float)(T * B);
    float carry = 0.f;
    float acc[3] = {0.f, 0.f, 0.f};
    // scan lanes keep vs of the row just above the current slab in a register: V_T for the first slab (vtrace.py:127)
    float above = 0.f;
    if (threadIdx.x < TC && c0 + threadIdx.x < B) above = a.value[T * B + c0 + threadIdx.x];
    for (long long hi = T; hi > 0; hi -= CHUNK) {
        const long long lo = hi > CHUNK ? hi - CHUNK : 0;
        const int rows = (int)(hi - lo);
        for (int i = threadIdx.x; i < rows * TC; i += NT) {
            const int r = i / TC, cc = i % TC;
            const long long c = c0 + cc;
            if (c < B) {
                const long long off = (lo + r) * B + c;
                const float is = ldg_stream(a.isw + off);
                const bool nan = is != is;  // torch.clamp keeps NaN, fminf would return the clip
                const float v = a.value[off], vn = a.value[off + B];
                const float rw = ldg_stream(a.reward + off);
                s_d[r][cc] = fmul(nan ? is : fminf(is, a.rho_clip), fsub(fadd(rw, fmul(a.gamma, vn)), v));
                s_f[r][cc] = fmul(a.gamma_lambda, nan ? is : fminf(is, a.c_clip));
                s_v[r][cc] = v;
                s_g[r][cc] = nan ? is : fminf(is, a.rho_pg_clip);
                s_r[r][cc] = rw;
                s_w[r][cc] = a.weight ? ldg_stream(a.weight + off) : 1.f;
                s_l[r][cc] = ldg_stream(a.lp_t + off);
                s_e[r][cc] = ldg_stream(a.ent + off);
            }
        }
        __syncthreads();
        if (threadIdx.x < TC && c0 + threadIdx.x < B) {
            const int cc = threadIdx.x;
            s_vs[rows][cc] = above;
            float vs = above;
            for (int r = rows - 1; r >= 0; --r) {
                carry = fadd(s_d[r][cc], fmul(s_f[r][cc], carry));
                vs = fadd(s_v[r][cc], carry);  // result[t] += item
                s_vs[r][cc] = vs;
            }
            above = vs;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < rows * TC; i += NT) {
            const int r = i / TC, cc = i % TC;
            const long long c = c0 + cc;
            if (c < B) {
                const long long off = (lo + r) * B + c;
                const float w = s_w[r][cc], v = s_v[r][cc];
                const float adv = fmul(s_g[r][cc], fsub(fadd(s_r[r][cc], fmul(a.gamma, s_vs[r + 1][cc])), v));
                const float dv = v - s_vs[r][cc];
                acc[0] += s_l[r][cc] * adv * w;
                acc[1] += dv * dv * w;
                acc[2] += s_e[r][cc] * w;
                stg_stream(a.isw + off, adv * w);               // coefficient of the policy-gradient term
                stg_stream(a.ent + off, 2.f * w * dv * inv_m);  // d value_loss / d V_t
            }
        }
        __syncthreads();
    }
    double tot[3];
    if (grid_sum<3, NT>(acc, tot, ws, 0) && threadIdx.x == 0) {
        const double m = (double)T * (double)B;
        a.out[0] = (float)(-tot[0] / m);
        a.out[1] = (float)(tot[1] / m);
        a.out[2] = (float)(tot[2] / m);
    }
}

// backward: grad z_j = g_pg*(-adv*w/M)*(1[j==a]-p_j) + g_ent*(w/M)*(-p_j*(logp_j+H)); grad V_t = g_val*dV, grad V_T = 0
template <int NT, int MODE>  // 0 staged thread/row, 1 direct thread/row, 2 warp/row
__global__ void __launch_bounds__(NT) vtrace_bwd_kernel(VtArgs a) {
    pdl_prologue();
    extern __shared__ __align__(16) float smem[];
    constexpr int L = (MODE == 2) ? 32 : 1;
    const int lane = (MODE == 2) ? (threadIdx.x & 31) : 0;
    const int N = a.N;
    const long long M = a.T * a.B;
    const float g_pg = a.g_pg ? *a.g_pg : 0.f, g_val = a.g_val ? *a.g_val : 0.f, g_ent = a.g_ent ? *a.g_ent : 0.f;
    const float inv_m = 1.f / (float)M;
    long long row0 = 0, row;
    int nflt = 0;
    const float* z;
    float* gz;
    if (MODE == 0) {
        row0 = (long long)blockIdx.x * NT;
        nflt = (int)min((long long)NT, M - row0) * N;
        stage_rows<NT>(smem, a.target + row0 * N, nflt, true);
        __syncthreads();
        row = row0 + threadIdx.x;
        z = smem + threadIdx.x * N;
        gz = smem + threadIdx.x * N;
    } else {
        row = (MODE == 2) ? (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5)
                          : (long long)blockIdx.x * NT + threadIdx.x;
        z = a.target + row * N;
        gz = a.grad_logit + row * N;
    }
    if (row < M) {
        const float w = a.weight ? a.weight[row] : 1.f;
        const int act = (int)a.action[row];
        float lse, ent;
        row_lse_entropy<L>([&](int j) { return z[j]; }, N, lane, lse, ent);
        const float c_act = g_pg * (-a.isw[row]) * inv_m;  // isw now holds adv*w
        const float c_ent = g_ent * w * inv_m;
        for (int j = lane; j < N; j += L) {
            const float lp = fmaxf(z[j] - lse, kF32Min);  // Categorical.entropy's clamp: 0 * finite at a -inf logit
            const float p = expf(lp);
            float gj = -c_act * p - c_ent * p * (lp + ent);
            if (j == act) gj += c_act;
            gz[j] = gj;
        }
        if (lane == 0) a.grad_value[row] = g_val * a.ent[row];  // ent now holds dV
    }
    // zero gradient for the bootstrap row V_T
    {
        const long long i = (long long)blockIdx.x * NT + threadIdx.x;  // gridDim.x * NT >= M >= B in every mode
        if (i < a.B) a.grad_value[M + i] = 0.f;
    }
    if (MODE == 0) {
        __syncthreads();
        float4* out4 = reinterpret_cast<float4*>(a.grad_logit + row0 * N);
        const int nv4 = nflt >> 2;
        for (int i = threadIdx.x; i < nv4; i += NT) stg_stream4(out4 + i, reinterpret_cast<const float4*>(smem)[i]);
        for (int i = (nv4 << 2) + threadIdx.x; i < nflt; i += NT) a.grad_logit[row0 * N + i] = smem[i];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// vtrace_error_continuous_action (ding/rl_utils/vtrace.py:139-212): Independent(Normal(mu, sigma)) policies.  Rows kernel ->
// the shared scan -> backward rows kernel (SURVEY section 8f rank 3).
// ---------------------------------------------------------------------------------------------------------------
struct VtcArgs {
    const float* mu_t;     // (M, D) target policy
    const float* sigma_t;
    const float* mu_b;     // (M, D) behaviour policy
    const float* sigma_b;
    const float* action;   // (M, D)
    const float* weight;   // nullable (M)
    long long M;
    int D;
    float* lp_t;           // (M) log pi(a)            | backward: unused
    float* isw;            // (M) importance weight    | backward: cpg = adv*w
    float* ent;            // (M) entropy              | backward: dV
    const float* g_pg;
    const float* g_val;
    const float* g_ent;
    float* grad_mu;
    float* grad_sigma;
    float* grad_value;     // (T+1, B)
    long long B;
};

__device__ __forceinline__ float vtc_logp(const float* mu, const float* sg, const float* ac, int D) {
    float lp = 0.f;
    for (int d = 0; d < D; ++d) {
        const float df = ac[d] - mu[d], s_ = sg[d];
        lp += -(df * df) / (2.f * s_ * s_) - logf(s_) - 0.9189385332046727f;  // Normal.log_prob
    }
    return lp;
}

__global__ void __launch_bounds__(256) vtc_rows_kernel(VtcArgs a) {
    pdl_prologue();
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < a.M; i += (long long)gridDim.x * 256) {
        const long long o = i * a.D;
        const float lp = vtc_logp(a.mu_t + o, a.sigma_t + o, a.action + o, a.D);
        const float lb = vtc_logp(a.mu_b + o, a.sigma_b + o, a.action + o, a.D);
        float e = 0.f;
        for (int d = 0; d < a.D; ++d) e += 1.4189385332046727f + logf(a.sigma_t[o + d]);  // Normal.entropy
        a.lp_t[i] = lp;
        a.isw[i] = expf(lp - lb);  // isw.py:49-53
        a.ent[i] = e;
    }
}

__global__ void __launch_bounds__(256) vtc_bwd_kernel(VtcArgs a) {
    pdl_prologue();
    const float g_pg = a.g_pg ? *a.g_pg : 0.f, g_val = a.g_val ? *a.g_val : 0.f, g_ent = a.g_ent ? *a.g_ent : 0.f;
    const float inv_m = 1.f / (float)a.M;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < a.M + a.B; i += (long long)gridDim.x * 256) {
        if (i >= a.M) {  // the bootstrap row V_T receives no gradient
            a.grad_value[i] = 0.f;
            continue;
        }
        const long long o = i * a.D;
        const float w = a.weight ? a.weight[i] : 1.f;
        const float c_lp = g_pg * (-a.isw[i]) * inv_m;  // d (-mean(lp * adv * w)) / d lp
        const float c_ent = g_ent * w * inv_m;
        for (int d = 0; d < a.D; ++d) {
            const float sd = a.sigma_t[o + d], df = a.action[o + d] - a.mu_t[o + d], inv = 1.f / sd;
            a.grad_mu[o + d] = c_lp * df * inv * inv;
            a.grad_sigma[o + d] = c_lp * (df * df * inv * inv * inv - inv) + c_ent * inv;
        }
        a.grad_value[i] = g_val * a.ent[i];
    }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_upgo_head_fwd(const float* logit, const long long* action, const float* mask, const float* rho,
                                    const float* ret, const float* value, long long TB, long long K, long long N,
                                    float* loss, float* adv_saved, float* grad_logit_unit, float* workspace,
                                    size_t workspace_bytes, void* stream) {
    if (TB <= 0 || K < 1 || N < 1 || !logit || !action || !rho || !ret || !value || !loss || !adv_saved || !workspace)
        return B200RL_ERR_ARG;
    UpgoArgs a{};
    a.logit = logit; a.action = action; a.mask = mask; a.rho = rho; a.ret = ret; a.value = value; a.TB = TB;
    a.K = (int)K; a.N = (int)N; a.loss = loss; a.adv_saved = adv_saved; a.grad_unit = grad_logit_unit;
    constexpr int NT = 128;
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int MAX_GRID = NUM_SMS * 16;
    if (N > 64) {
        int grid = div_up(TB, NT / 32);
        if (grid > MAX_GRID) grid = MAX_GRID;
        if (!ws_partials_fit((long long)(grid), workspace_bytes)) return B200RL_ERR_WORKSPACE;
        return launch_k(upgo_fwd_kernel<NT, 32>, grid, NT, 0, st, a, workspace);
    }
    int grid = div_up(TB, NT);
    if (grid > MAX_GRID) grid = MAX_GRID;
    if (!ws_partials_fit((long long)(grid), workspace_bytes)) return B200RL_ERR_WORKSPACE;
    return launch_k(upgo_fwd_kernel<NT, 1>, grid, NT, 0, st, a, workspace);
}

extern "C" int b200rl_upgo_head_bwd(const float* logit, const long long* action, const float* mask,
                                    const float* adv_saved, const float* g_loss, long long TB, long long K,
                                    long long N, int skip_if_unit, float* grad_logit, void* stream) {
    if (TB <= 0 || K < 1 || N < 1 || !logit || !action || !adv_saved || !grad_logit) return B200RL_ERR_ARG;
    UpgoArgs a{};
    a.logit = logit; a.action = action; a.mask = mask; a.adv_saved = const_cast<float*>(adv_saved); a.TB = TB;
    a.K = (int)K; a.N = (int)N; a.g_loss = g_loss; a.grad_logit = grad_logit; a.skip_if_unit = skip_if_unit;
    constexpr int NT = 128;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = N > 64 ? div_up(TB * K, NT / 32) : div_up(TB * K, NT);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    if (N > 64) return launch_k(upgo_bwd_kernel<NT, 32>, grid, NT, 0, st, a);
    return launch_k(upgo_bwd_kernel<NT, 1>, grid, NT, 0, st, a);
}

extern "C" int b200rl_tb_cross_entropy_fwd(const float* logit, const long long* action, const float* mask, long long TB,
                                           long long K, long long N, float* ce, void* stream) {
    if (TB <= 0 || K < 1 || N < 1 || !logit || !action || !ce) return B200RL_ERR_ARG;
    constexpr int NT = 128;
    cudaStream_t st = (cudaStream_t)stream;
    if (N > 64) return launch_k(tbce_fwd_kernel<NT, 32>, div_up(TB, NT / 32), NT, 0, st, logit, action, mask, TB, (int)K, (int)N, ce);
    return launch_k(tbce_fwd_kernel<NT, 1>, div_up(TB, NT), NT, 0, st, logit, action, mask, TB, (int)K, (int)N, ce);
}

extern "C" int b200rl_tb_cross_entropy_bwd(const float* logit, const long long* action, const float* mask,
                                           const float* g_ce, long long TB, long long K, long long N, float* grad_logit,
                                           void* stream) {
    if (TB <= 0 || K < 1 || N < 1 || !logit || !action || !g_ce || !grad_logit) return B200RL_ERR_ARG;
    constexpr int NT = 128;
    cudaStream_t st = (cudaStream_t)stream;
    if (N > 64) return launch_k(tbce_bwd_kernel<NT, 32>, div_up(TB * K, NT / 32), NT, 0, st, logit, action, mask, g_ce, TB, (int)K, (int)N, grad_logit);
    return launch_k(tbce_bwd_kernel<NT, 1>, div_up(TB * K, NT), NT, 0, st, logit, action, mask, g_ce, TB, (int)K, (int)N, grad_logit);
}

// ===============================================================================================================
// V-trace row kernels on the persistent TMA pipeline of ppo.cu (producer warp + 4 consumer warps, 3-stage ring of
// 1-D bulk copies, no CTA-wide barrier in the loop).  Used when N <= 32 and every tensor is 16-byte aligned.
//   vt_rows_tile_kernel : stage = target logits | behaviour logits | actions  ->  lp(a), importance weight, entropy
//   vt_bwd_tile_kernel  : stage = target logits | actions | adv*w | dV [| w]  ->  gradient rows through shared memory
//                         and per-warp TMA bulk stores, d/dV straight from registers
// ===============================================================================================================
constexpr int VT_R = PPO_CT;  // rows per tile (one per consumer thread)

template <int NC>
__global__ void __launch_bounds__(PPO_THREADS) vt_rows_tile_kernel(VtArgs a) {
    pdl_prologue();
    extern __shared__ __align__(128) unsigned char smem[];
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const long long M = a.T * a.B;
    const int logit_bytes = VT_R * N * 4;
    const int off_beh = logit_bytes, off_act = 2 * logit_bytes;
    const int stage_bytes = (2 * logit_bytes + VT_R * 8 + 127) & ~127;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + PPO_STAGES * stage_bytes);
    uint64_t* empty = full + PPO_STAGES;
    const long long n_full = M / VT_R;
    const int tail_rows = (int)(M - n_full * VT_R);
    const long long n_tiles = n_full + (tail_rows ? 1 : 0);
    const int my_n = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;
    if (tid == 0) {
        for (int s = 0; s < PPO_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], PPO_CW);
        }
        mbar_fence_init();
    }
    __syncthreads();
    if (wid == PPO_CW) {
        if (lane == 0) {
            for (int i = 0; i < my_n; ++i) {
                const long long t = blockIdx.x + (long long)i * gridDim.x;
                if (t >= n_full) break;
                const int sg = i % PPO_STAGES;
                if (i >= PPO_STAGES) mbar_wait(&empty[sg], (uint32_t)(((i / PPO_STAGES) - 1) & 1));
                const long long row0 = t * VT_R;
                unsigned char* st = smem + sg * stage_bytes;
                mbar_expect_tx(&full[sg], (uint32_t)(2 * logit_bytes + VT_R * 8));
                tma_load_1d(st, a.target + row0 * N, logit_bytes, &full[sg]);
                tma_load_1d(st + off_beh, a.behaviour + row0 * N, logit_bytes, &full[sg]);
                tma_load_1d(st + off_act, a.action + row0, VT_R * 8, &full[sg]);
            }
        }
        return;
    }
    for (int i = 0; i < my_n; ++i) {
        const long long t = blockIdx.x + (long long)i * gridDim.x;
        const long long row0 = t * VT_R;
        const int sg = i % PPO_STAGES;
        unsigned char* st = smem + sg * stage_bytes;
        const bool full_tile = t < n_full;
        if (full_tile) {
            mbar_wait(&full[sg], (uint32_t)((i / PPO_STAGES) & 1));
        } else if (tid < tail_rows) {
            for (int k = 0; k < N; ++k) {
                reinterpret_cast<float*>(st)[tid * N + k] = a.target[(row0 + tid) * N + k];
                reinterpret_cast<float*>(st + off_beh)[tid * N + k] = a.behaviour[(row0 + tid) * N + k];
            }
            reinterpret_cast<long long*>(st + off_act)[tid] = a.action[row0 + tid];
        }
        if (full_tile || tid < tail_rows) {
            const float* zt = reinterpret_cast<const float*>(st) + tid * N;
            const float* zb = reinterpret_cast<const float*>(st + off_beh) + tid * N;
            const int act = (int)reinterpret_cast<const long long*>(st + off_act)[tid];
            constexpr int NR = NC ? NC : 1;
            float m = kF32Min, s = 0.f, u2 = 0.f, mb = kF32Min, sb = 0.f;
            if (NC) {
                float tt[NR], tb[NR];
                load_row<NR>(zt, tt);
                load_row<NR>(zb, tb);
#pragma unroll
                for (int j = 0; j < NR; ++j) { m = fmaxf(m, tt[j]); mb = fmaxf(mb, tb[j]); }
                const float m2 = m * kLog2e, mb2 = mb * kLog2e;
#pragma unroll
                for (int j = 0; j < NR; ++j) {
                    const float x = fmaxf(fmaf(tt[j], kLog2e, -m2), kF32Min);
                    const float e = ex2f_(x);
                    s += e;
                    u2 = fmaf(e, x, u2);
                    sb += ex2f_(fmaf(tb[j], kLog2e, -mb2));
                }
            } else {
                for (int j = 0; j < N; ++j) { m = fmaxf(m, zt[j]); mb = fmaxf(mb, zb[j]); }
                const float m2 = m * kLog2e, mb2 = mb * kLog2e;
                for (int j = 0; j < N; ++j) {
                    const float x = fmaxf(fmaf(zt[j], kLog2e, -m2), kF32Min);
                    const float e = ex2f_(x);
                    s += e;
                    u2 = fmaf(e, x, u2);
                    sb += ex2f_(fmaf(zb[j], kLog2e, -mb2));
                }
            }
            const float l2s = lg2f_(s);
            const float lp_t = (zt[act] - m) - l2s * kLn2;
            const float lp_b = (zb[act] - mb) - lg2f_(sb) * kLn2;
            a.lp_t[row0 + tid] = lp_t;
            a.isw[row0 + tid] = ex2f_((lp_t - lp_b) * kLog2e);
            a.ent[row0 + tid] = (l2s - u2 * rcpf_(s)) * kLn2;
        }
        if (full_tile) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[sg]);
        }
    }
}

template <int NC>
__global__ void __launch_bounds__(PPO_THREADS) vt_bwd_tile_kernel(VtArgs a) {
    pdl_prologue();
    extern __shared__ __align__(128) unsigned char smem[];
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const long long M = a.T * a.B;
    const bool has_w = a.weight != nullptr;
    const int logit_bytes = VT_R * N * 4;
    const int off_act = logit_bytes, off_c = off_act + VT_R * 8, off_dv = off_c + VT_R * 4, off_w = off_dv + VT_R * 4;
    const int tx_bytes = off_w + (has_w ? VT_R * 4 : 0);
    const int stage_bytes = (tx_bytes + 127) & ~127;
    const int warp_out_bytes = 32 * N * 4;
    unsigned char* outbuf = smem + PPO_STAGES * stage_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + 2 * logit_bytes);
    uint64_t* empty = full + PPO_STAGES;
    const float g_pg = a.g_pg ? *a.g_pg : 0.f, g_val = a.g_val ? *a.g_val : 0.f, g_ent = a.g_ent ? *a.g_ent : 0.f;
    const float inv_m = 1.f / (float)M;
    {   // bootstrap row V_T receives no gradient (value[:-1], vtrace.py:134)
        const long long i = (long long)blockIdx.x * PPO_THREADS + tid;
        for (long long c = i; c < a.B; c += (long long)gridDim.x * PPO_THREADS) a.grad_value[M + c] = 0.f;
    }
    const long long n_full = M / VT_R;
    const int tail_rows = (int)(M - n_full * VT_R);
    const long long n_tiles = n_full + (tail_rows ? 1 : 0);
    const int my_n = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;
    if (tid == 0) {
        for (int s = 0; s < PPO_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], PPO_CW);
        }
        mbar_fence_init();
    }
    __syncthreads();
    if (wid == PPO_CW) {
        if (lane == 0) {
            for (int i = 0; i < my_n; ++i) {
                const long long t = blockIdx.x + (long long)i * gridDim.x;
                if (t >= n_full) break;
                const int sg = i % PPO_STAGES;
                if (i >= PPO_STAGES) mbar_wait(&empty[sg], (uint32_t)(((i / PPO_STAGES) - 1) & 1));
                const long long row0 = t * VT_R;
                unsigned char* st = smem + sg * stage_bytes;
                mbar_expect_tx(&full[sg], (uint32_t)tx_bytes);
                tma_load_1d(st, a.target + row0 * N, logit_bytes, &full[sg]);
                tma_load_1d(st + off_act, a.action + row0, VT_R * 8, &full[sg]);
                tma_load_1d(st + off_c, a.isw + row0, VT_R * 4, &full[sg]);   // adv*w
                tma_load_1d(st + off_dv, a.ent + row0, VT_R * 4, &full[sg]);  // dV
                if (has_w) tma_load_1d(st + off_w, a.weight + row0, VT_R * 4, &full[sg]);
            }
        }
        return;
    }
    for (int i = 0; i < my_n; ++i) {
        const long long t = blockIdx.x + (long long)i * gridDim.x;
        const long long row0 = t * VT_R;
        const int sg = i % PPO_STAGES;
        unsigned char* st = smem + sg * stage_bytes;
        const bool full_tile = t < n_full;
        if (full_tile) {
            mbar_wait(&full[sg], (uint32_t)((i / PPO_STAGES) & 1));
        } else if (tid < tail_rows) {
            for (int k = 0; k < N; ++k) reinterpret_cast<float*>(st)[tid * N + k] = a.target[(row0 + tid) * N + k];
            reinterpret_cast<long long*>(st + off_act)[tid] = a.action[row0 + tid];
            reinterpret_cast<float*>(st + off_c)[tid] = a.isw[row0 + tid];
            reinterpret_cast<float*>(st + off_dv)[tid] = a.ent[row0 + tid];
            if (has_w) reinterpret_cast<float*>(st + off_w)[tid] = a.weight[row0 + tid];
        }
        float* wbuf = reinterpret_cast<float*>(outbuf + (wid * 2 + (i & 1)) * warp_out_bytes);
        if (full_tile || tid < tail_rows) {
            const float* z = reinterpret_cast<const float*>(st) + tid * N;
            const int act = (int)reinterpret_cast<const long long*>(st + off_act)[tid];
            const float cpg = reinterpret_cast<const float*>(st + off_c)[tid];
            const float dv = reinterpret_cast<const float*>(st + off_dv)[tid];
            const float w = has_w ? reinterpret_cast<const float*>(st + off_w)[tid] : 1.f;
            constexpr int NR = NC ? NC : 1;
            float tn[NR], en[NR];
            float m = kF32Min, s = 0.f, u2 = 0.f;
            if (NC) {
                load_row<NR>(z, tn);
#pragma unroll
                for (int j = 0; j < NR; ++j) m = fmaxf(m, tn[j]);
                const float m2 = m * kLog2e;
#pragma unroll
                for (int j = 0; j < NR; ++j) {
                    tn[j] = fmaxf(fmaf(tn[j], kLog2e, -m2), kT2Min);
                    en[j] = ex2f_(tn[j]);
                    s += en[j];
                    u2 = fmaf(en[j], tn[j], u2);
                }
            } else {
                for (int j = 0; j < N; ++j) m = fmaxf(m, z[j]);
                const float m2 = m * kLog2e;
                for (int j = 0; j < N; ++j) {
                    const float x = fmaxf(fmaf(z[j], kLog2e, -m2), kT2Min);
                    const float e = ex2f_(x);
                    s += e;
                    u2 = fmaf(e, x, u2);
                }
            }
            const float l2s = lg2f_(s), inv_sum = rcpf_(s);
            const float log_s = l2s * kLn2, ent = (l2s - u2 * inv_sum) * kLn2;
            // grad z_j = c_act*(1[j==a]-p_j) - c_ent*p_j*(logp_j + H) = p_j*(k0 - k1*t_j) + 1[j==a]*c_act
            const float c_act = g_pg * (-cpg) * inv_m, c_ent = g_ent * w * inv_m;
            const float k0 = -c_act - c_ent * (ent - log_s), k1 = c_ent * kLn2;
            float* gr = full_tile ? wbuf + lane * N : a.grad_logit + (row0 + tid) * N;
            if (NC) {
                float gj[NR];
#pragma unroll
                for (int j = 0; j < NR; ++j) {
                    gj[j] = (en[j] * inv_sum) * fmaf(-k1, tn[j], k0);
                    if (j == act) gj[j] += c_act;
                }
                store_row<NR>(gr, gj);
            } else {
                const float m2 = m * kLog2e;
                for (int j = 0; j < N; ++j) {
                    const float x = fmaxf(fmaf(z[j], kLog2e, -m2), kT2Min);
                    float g = (ex2f_(x) * inv_sum) * fmaf(-k1, x, k0);
                    if (j == act) g += c_act;
                    gr[j] = g;
                }
            }
            a.grad_value[row0 + tid] = g_val * dv;
        }
        if (full_tile) {
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) {
                tma_store_1d(a.grad_logit + (row0 + wid * 32) * N, wbuf, warp_out_bytes);
                tma_store_commit();
                tma_store_wait_read<1>();
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[sg]);
        }
    }
    if (lane == 0) tma_store_wait_read<0>();
}

template <int NC, bool BWD>
static int launch_vt_tile(const VtArgs& a, cudaStream_t st) {
    const int N = a.N;
    const int logit_bytes = VT_R * N * 4;
    size_t smem;
    if (BWD) {
        const int tx = logit_bytes + VT_R * 8 + VT_R * 4 * 2 + (a.weight ? VT_R * 4 : 0);
        smem = (size_t)PPO_STAGES * ((tx + 127) & ~127) + 2 * logit_bytes + 2 * PPO_STAGES * sizeof(uint64_t);
    } else {
        smem = (size_t)PPO_STAGES * ((2 * logit_bytes + VT_R * 8 + 127) & ~127) + 2 * PPO_STAGES * sizeof(uint64_t);
    }
    constexpr void (*kern)(VtArgs) = BWD ? vt_bwd_tile_kernel<NC> : vt_rows_tile_kernel<NC>;
    if (smem > 227 * 1024) return B200RL_ERR_ARG;
    int sm_count, per_sm;
    if (int rc = resident_ctas<kern>(PPO_THREADS, smem, sm_count, per_sm)) return rc;
    if (per_sm > 6) per_sm = 6;
    const long long n_tiles = (a.T * a.B + VT_R - 1) / VT_R;
    long long grid = (long long)sm_count * per_sm;
    if (grid > n_tiles) grid = n_tiles;
    return launch_k(kern, (int)grid, PPO_THREADS, smem, st, a);
}

template <bool BWD>
static int dispatch_vt_tile(const VtArgs& a, cudaStream_t st) {
    return with_nc(a.N, [&](auto nc) { return launch_vt_tile<nc, BWD>(a, st); });
}

static bool vt_tile_ok(const VtArgs& a, bool bwd) {
    bool al = aligned16(a.target) && aligned16(a.action) && aligned16(a.isw) && aligned16(a.ent) &&
              (!a.weight || aligned16(a.weight));
    if (bwd) al = al && aligned16(a.grad_logit);
    else al = al && aligned16(a.behaviour);
    return al && a.N <= 32;
}

// the column-tile scan that turns (log pi(a), importance weight, entropy) rows into vs / advantages / losses / gradient
// coefficients: shared by the discrete and the continuous head
static int launch_vt_scan(const VtArgs& a, float* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (a.B >= 16 * 2 * NUM_SMS) {
        if (!ws_partials_fit((long long)(3 * div_up(a.B, 16)), workspace_bytes)) return B200RL_ERR_WORKSPACE;
        return launch_k(vtrace_scan_kernel<16, 256, 64>, div_up(a.B, 16), 256, 0, st, a, workspace);
    }
    if (!ws_partials_fit((long long)(3 * div_up(a.B, 8)), workspace_bytes)) return B200RL_ERR_WORKSPACE;
    return launch_k(vtrace_scan_kernel<8, 64, 64>, div_up(a.B, 8), 64, 0, st, a, workspace);
}

static int vt_mode(const VtArgs& a) {
    const bool al = aligned16(a.target) && aligned16(a.behaviour) && (!a.grad_logit || aligned16(a.grad_logit));
    if (a.N <= 32 && al) return 0;
    if (a.N <= 64) return 1;
    return 2;
}

extern "C" int b200rl_vtrace_fwd(const float* target_output, const float* behaviour_output, const long long* action,
                                 const float* value, const float* reward, const float* weight, long long T,
                                 long long B, long long N, double gamma, double lambda_, double rho_clip_ratio,
                                 double c_clip_ratio, double rho_pg_clip_ratio, float* out3, float* lp_saved,
                                 float* cpg_saved, float* dv_saved, float* workspace, size_t workspace_bytes,
                                 void* stream) {
    if (T <= 0 || B <= 0 || N < 1 || !target_output || !behaviour_output || !action || !value || !reward || !out3 ||
        !lp_saved || !cpg_saved || !dv_saved || !workspace)
        return B200RL_ERR_ARG;
    VtArgs a{};
    a.target = target_output; a.behaviour = behaviour_output; a.action = action; a.value = value; a.reward = reward;
    a.weight = weight; a.T = T; a.B = B; a.N = (int)N; a.gamma = (float)gamma;
    a.gamma_lambda = (float)(gamma * lambda_);  // `factor = gamma * lambda_` in python double, vtrace.py:23
    a.rho_clip = (float)rho_clip_ratio; a.c_clip = (float)c_clip_ratio; a.rho_pg_clip = (float)rho_pg_clip_ratio;
    a.lp_t = lp_saved; a.isw = cpg_saved; a.ent = dv_saved; a.out = out3;
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int NT = 128;
    const long long M = T * B;
    const int mode = vt_mode(a);
    int rc;
    if (vt_tile_ok(a, false))
        rc = dispatch_vt_tile<false>(a, st);
    else if (mode == 0)
        rc = launch_k(vtrace_rows_kernel<NT, true>, div_up(M, NT), NT, (size_t)2 * NT * a.N * sizeof(float), st, a);
    else if (mode == 1)
        rc = launch_k(vtrace_rows_kernel<NT, false>, div_up(M, NT), NT, 0, st, a);
    else
        rc = launch_k(vtrace_rows_warp_kernel<NT>, div_up(M, NT / 32), NT, 0, st, a);
    if (rc) return rc;
    return launch_vt_scan(a, workspace, workspace_bytes, st);
}

extern "C" int b200rl_vtrace_bwd(const float* target_output, const long long* action, const float* weight,
                                 const float* cpg_saved, const float* dv_saved, const float* g_policy,
                                 const float* g_value, const float* g_entropy, long long T, long long B, long long N,
                                 float* grad_target_output, float* grad_value, void* stream) {
    if (T <= 0 || B <= 0 || N < 1 || !target_output || !action || !cpg_saved || !dv_saved || !grad_target_output ||
        !grad_value)
        return B200RL_ERR_ARG;
    VtArgs a{};
    a.target = target_output; a.behaviour = target_output; a.action = action; a.weight = weight; a.T = T; a.B = B;
    a.N = (int)N; a.isw = const_cast<float*>(cpg_saved); a.ent = const_cast<float*>(dv_saved);
    a.g_pg = g_policy; a.g_val = g_value; a.g_ent = g_entropy; a.grad_logit = grad_target_output;
    a.grad_value = grad_value;
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int NT = 128;
    const long long M = T * B;
    const int mode = vt_mode(a);
    if (vt_tile_ok(a, true)) return dispatch_vt_tile<true>(a, st);
    if (mode == 0) return launch_k(vtrace_bwd_kernel<NT, 0>, div_up(M, NT), NT, (size_t)NT * a.N * sizeof(float), st, a);
    if (mode == 1) return launch_k(vtrace_bwd_kernel<NT, 1>, div_up(M, NT), NT, 0, st, a);
    return launch_k(vtrace_bwd_kernel<NT, 2>, div_up(M, NT / 32), NT, 0, st, a);
}

extern "C" int b200rl_vtrace_continuous_fwd(const float* mu_target, const float* sigma_target, const float* mu_behaviour,
                                            const float* sigma_behaviour, const float* action, const float* value,
                                            const float* reward, const float* weight, long long T, long long B, long long D,
                                            double gamma, double lambda_, double rho_clip_ratio, double c_clip_ratio,
                                            double rho_pg_clip_ratio, float* out3, float* lp_saved, float* cpg_saved,
                                            float* dv_saved, float* workspace, size_t workspace_bytes, void* stream) {
    if (T <= 0 || B <= 0 || D < 1 || !mu_target || !sigma_target || !mu_behaviour || !sigma_behaviour || !action || !value ||
        !reward || !out3 || !lp_saved || !cpg_saved || !dv_saved || !workspace)
        return B200RL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    VtcArgs r{};
    r.mu_t = mu_target; r.sigma_t = sigma_target; r.mu_b = mu_behaviour; r.sigma_b = sigma_behaviour; r.action = action;
    r.M = T * B; r.D = (int)D; r.lp_t = lp_saved; r.isw = cpg_saved; r.ent = dv_saved;
    long long grid = div_up(r.M, 256);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    if (int rc = launch_k(vtc_rows_kernel, (int)grid, 256, 0, st, r)) return rc;
    VtArgs a{};
    a.value = value; a.reward = reward; a.weight = weight; a.T = T; a.B = B; a.N = (int)D; a.gamma = (float)gamma;
    a.gamma_lambda = (float)(gamma * lambda_);
    a.rho_clip = (float)rho_clip_ratio; a.c_clip = (float)c_clip_ratio; a.rho_pg_clip = (float)rho_pg_clip_ratio;
    a.lp_t = lp_saved; a.isw = cpg_saved; a.ent = dv_saved; a.out = out3;
    return launch_vt_scan(a, workspace, workspace_bytes, st);
}

extern "C" int b200rl_vtrace_continuous_bwd(const float* mu_target, const float* sigma_target, const float* action,
                                            const float* weight, const float* cpg_saved, const float* dv_saved,
                                            const float* g_policy, const float* g_value, const float* g_entropy, long long T,
                                            long long B, long long D, float* grad_mu, float* grad_sigma, float* grad_value,
                                            void* stream) {
    if (T <= 0 || B <= 0 || D < 1 || !mu_target || !sigma_target || !action || !cpg_saved || !dv_saved || !grad_mu ||
        !grad_sigma || !grad_value)
        return B200RL_ERR_ARG;
    VtcArgs r{};
    r.mu_t = mu_target; r.sigma_t = sigma_target; r.action = action; r.weight = weight; r.M = T * B; r.B = B; r.D = (int)D;
    r.isw = const_cast<float*>(cpg_saved); r.ent = const_cast<float*>(dv_saved);
    r.g_pg = g_policy; r.g_val = g_value; r.g_ent = g_entropy; r.grad_mu = grad_mu; r.grad_sigma = grad_sigma;
    r.grad_value = grad_value;
    long long grid = div_up(r.M + B, 256);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    return launch_k(vtc_bwd_kernel, (int)grid, 256, 0, (cudaStream_t)stream, r);
}
