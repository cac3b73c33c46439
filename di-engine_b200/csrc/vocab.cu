// Vocabulary-scale token losses of the language-model policy-gradient family, on fp32 or bf16 logits:
//   grpo_policy_error                 ding/rl_utils/grpo.py             clipped ratio loss + beta * k3 KL to the reference policy
//   rloo_policy_error                 ding/rl_utils/rloo.py             clipped ratio loss, leave-one-out advantage from reward (K, B')
//   naive / efficient / less_efficient_method   ding/rl_utils/log_prob_utils.py   per-token log p(a) and its backward
//
// vocab_rows_kernel<T, MODE>: persistent CTAs of VOCAB_NT threads, each owning one token row of V logits at a time
// (row += gridDim.x).  Per row, in ONE streaming pass over every logit tensor of the call (16-byte vector loads, all
// streams' loads of an iteration in flight together), an online max / sum of exp in fp32 per tensor gives
// logsumexp = max + log(sum exp(z - max)) with torch's rule for an infinite max (treated as 0); the gathered z[a] gives
// lp = z[a] - logsumexp.  The row epilogue (thread 0) runs the token head (token_head below, in the reference's operation
// order) and forms c = d loss / d lp_new for a unit upstream gradient; the CTA then writes
// d loss / d logit_new[row] = c * (onehot(a) - softmax(logit_new[row])) in T.  MODE = LOGP writes lp and logsumexp only;
// MODE = BWD applies a per-row coefficient g * coef[row] to (onehot - softmax) -- the backward of the log-prob methods, and
// of the GRPO / RLOO launch when the upstream gradient is not the unit one the forward launch assumed.
//
// Traffic floor per token row: every logit read once plus the gradient written once, (3 + 1) * V * sizeof(T) for GRPO and
// (2 + 1) * V * sizeof(T) for RLOO; per-row side data (action, weight, lse, coefficient) is O(1) per row.
//
// The softmax of the gradient needs logit_new a second time.  The forward launch keeps the row in dynamic shared memory
// as it streams it, up to VOCAB_SMEM_CAP bytes (all of V = 32k in fp32 or V = 64k in bf16).  A longer row (bf16
// V = 152 064 is 304 KB) keeps its first VOCAB_SMEM_CAP bytes there and reads the rest back from L2 right after the
// same CTA streamed it: such a row runs one CTA per SM, so the bytes to re-read across the GPU are at most 132 * 84 KB
// = 11 MB, a fifth of the H100's 50 MB L2, and the other streams are loaded evict-first so they do not push it out.
// Chosen over splitting the row across a thread-block cluster because it keeps one code path for every V: a cluster
// split needs a second, DSMEM-level max / sum combine and a cluster size chosen per V, for the 28 % of the row that
// the L2 serves here.  The L2 holds the re-read only while 132 * (V * sizeof(T) - 220 KB) stays well below its 50 MB:
// up to about V = 190k in bf16 and V = 95k in fp32.  Past that (e.g. fp32 V = 152 064: 388 KB re-read per row, 51 MB
// across the GPU) part of the second read of logit_new goes to HBM and the call moves up to 5 * V * sizeof(T) bytes per
// row (GRPO) instead of the floor.
//
// The loss head on a custom log_prob_fn's (B, S) output is a second, small kernel (token_head_kernel below): it reads no
// logits, so it shares the head arithmetic (token_head) but none of the row machinery.
//
// Loss sums (loss, approx_kl, clipfrac): per-CTA partials (grid_store_partials) added in a fixed order by
// finalize_sums_kernel -- deterministic, no atomics, no host sync.
//
// PPO on token rows (ppo_policy_error / the policy part of ppo_error, ding/rl_utils/ppo.py:143-230, at (B, S, V)): MODE =
// VM_PPO + PPO_ENT (entropy bonus) + PPO_KL (logit_pretrained given), so the common RLHF call (no entropy, 2 or 3 streams)
// carries neither the entropy accumulator nor the third stream.  Next to logit_new's online max / sum of exp the pass keeps
// t = sum e^(z - r) * max(z - r, -FLT_MAX) (r the running max, rescaled with it like s), so H = log s - t / s reuses the
// exponentials already taken.  The row epilogue runs surrogate / kl_term (ppo_math.cuh) and, for the upstream gradients
// the call site expects (g_pol, g_ent, g_kl: its device-resident record), writes
// d / d logit_new = c_act * (onehot(a) - p) - c_ent * p * (log p + H), c_act = g_pol * (-w / M) * dsel * r + g_kl * dk / M,
// c_ent = g_ent * w / M (M rows).  Saved per row: lse, H (entropy only) and the unit coefficients (-w / M) * dsel * r and
// dk / M, from which VM_PPO_BWD recomputes the gradient for the actual upstream gradients (one read of logit_new, one
// write) -- unless they are the ones the forward used, in which case it returns at once on the device.  Loss sums:
// policy, entropy, kl, approx_kl, clipfrac, all over M.  Traffic: (3 + 1) * V * sizeof(T) per row with logit_pretrained,
// (2 + 1) without -- the same streams and the same L2 re-read of logit_new as GRPO / RLOO.
//
// A2C on token rows (a2c_error, ding/rl_utils/a2c.py:10-44, at (B, S, V) with a per-token value head): MODE = VM_A2C
// streams logit_new alone (NR = 1) with the entropy accumulator always on, and keeps the row in shared memory for the
// gradient's softmax as the other loss modes do.  The row epilogue follows the reference's order: lp = z[a] - lse,
// H, dv = return_ - value, partials -lp * adv * w, dv^2 * w, H * w (w = 1 without weight), all three means over M rows.
// For the expected upstream gradients (g_pol, g_val, g_ent: the call site's record) it writes
// d / d logit_new = c * (onehot(a) - p) - c_ent * p * (log p + H), c = g_pol * (-adv * w / M), c_ent = g_ent * w / M,
// and d / d value = g_val * (-2 * w * dv / M) in fp32.  Saved per row: lse, H, the unit coefficients -adv * w / M and
// -2 * w * dv / M.  The backward is VM_PPO_BWD + PPO_ENT + PPO_VAL, the PPO backward pass with the value slot: it returns
// at once when all three upstream gradients are the forward's, rewrites only d / d value (O(1) per row) when just g_val
// differs, and otherwise recomputes both.  Traffic: (1 + 1) * V * sizeof(T) per row, plus O(1) per row -- logit_new read
// once, its gradient written once, with the same L2 re-read of logit_new past VOCAB_SMEM_CAP.
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200rl.h"
#include "common.cuh"
#include "ppo_math.cuh"

namespace b200rl {

constexpr int VOCAB_NT = 512;
constexpr int VOCAB_HEAD_NT = 256;
constexpr int VOCAB_SMEM_CAP = 220 * 1024;  // dynamic shared memory for the cached part of logit_new (227 KB opt-in max)
constexpr int VM_GRPO = 0, VM_RLOO = 1, VM_LOGP = 2, VM_BWD = 3;
constexpr int VM_PPO = 4, VM_PPO_BWD = 8, PPO_ENT = 1, PPO_KL = 2;  // VM_PPO + flags: 4..7; VM_PPO_BWD + PPO_ENT: 8, 9
// A2C: forward 12; backward VM_PPO_BWD + PPO_ENT + PPO_VAL = 11 (the PPO backward with the value slot)
constexpr int PPO_VAL = 2, VM_A2C = 12;
constexpr float kL2E = 1.4426950408889634f;

// 16-byte vectors of T, widened to fp32
template <class T>
struct VecT;
template <>
struct VecT<float> {
    static constexpr int W = 4;
    static __device__ __forceinline__ void unpack(uint4 u, float (&x)[4]) {
        x[0] = __uint_as_float(u.x); x[1] = __uint_as_float(u.y); x[2] = __uint_as_float(u.z); x[3] = __uint_as_float(u.w);
    }
    static __device__ __forceinline__ uint4 pack(const float (&x)[4]) {
        return make_uint4(__float_as_uint(x[0]), __float_as_uint(x[1]), __float_as_uint(x[2]), __float_as_uint(x[3]));
    }
    static __device__ __forceinline__ float to_f(float v) { return v; }
    static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <>
struct VecT<__nv_bfloat16> {
    static constexpr int W = 8;
    static __device__ __forceinline__ void unpack(uint4 u, float (&x)[8]) {
        const unsigned int w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            x[2 * i] = __uint_as_float(w[i] << 16);
            x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
    static __device__ __forceinline__ uint4 pack(const float (&x)[8]) {
        unsigned int w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __nv_bfloat162 h = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
            w[i] = *reinterpret_cast<unsigned int*>(&h);
        }
        return make_uint4(w[0], w[1], w[2], w[3]);
    }
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// torch's logsumexp takes an infinite maximum as 0
__device__ __forceinline__ float lse_ref(float m) { return fabsf(m) == INFINITY ? 0.f : m; }

// e^d: exp2f(d * log2 e), or expf(d) where the entropy accumulator takes it (EXPF, see mst_add), so that every logit
// stream of a kernel forms its logsumexp with the same arithmetic (bit-identical streams give a ratio of exactly 1)
template <bool EXPF>
__device__ __forceinline__ float exp_of(float d) { return EXPF ? expf(d) : exp2f(d * kL2E); }

// online (max, sum exp(z - lse_ref(max))) over n values
template <int N, bool EXPF = false>
__device__ __forceinline__ void ms_add(float& m, float& s, const float (&x)[N]) {
    float mc = x[0];
#pragma unroll
    for (int i = 1; i < N; ++i) mc = fmaxf(mc, x[i]);
    if (mc > m) {
        if (s != 0.f) s *= exp_of<EXPF>(lse_ref(m) - lse_ref(mc));
        m = mc;
    }
    const float r = lse_ref(m);
    float e[N];
#pragma unroll
    for (int i = 0; i < N; ++i) e[i] = exp_of<EXPF>(x[i] - r);
    // pairwise within the vector, then one add to the running sum: a thread's sequential chain over a 152k-entry row is
    // N times shorter, and so is its fp32 rounding
#pragma unroll
    for (int w = 1; w < N; w *= 2)
#pragma unroll
        for (int i = 0; i + w < N; i += 2 * w) e[i] += e[i + w];
    s += e[0];
}

template <bool EXPF = false>
__device__ __forceinline__ void ms_merge(float& m, float& s, float m2, float s2) {
    if (m2 > m) {
        const float tm = m, ts = s;
        m = m2; s = s2; m2 = tm; s2 = ts;
    }
    if (s2 != 0.f) s += s2 * exp_of<EXPF>(lse_ref(m2) - lse_ref(m));
}

// ms_add with the entropy accumulator t = sum e^(z - r) * max(z - r, -FLT_MAX), r = lse_ref(max): a new max r' rescales
// it as t <- alpha * (t + s * (r - r')), alpha = e^(r - r'), and -inf logits add 0 (Categorical.entropy's clamp).  The
// exponentials here are expf, not exp2f((z - r) * log2 e): fp32 log2 e is off by 1.3e-8 relative, so every term with
// z - r ~ -50 carries the same ~7e-7 relative error, which does not average out and is all of H on a peaked row; the
// other logit streams of these kernels (ms_add / ms_merge with EXPF) take the same exponentials
template <int N>
__device__ __forceinline__ void mst_add(float& m, float& s, float& t, const float (&x)[N]) {
    float mc = x[0];
#pragma unroll
    for (int i = 1; i < N; ++i) mc = fmaxf(mc, x[i]);
    if (mc > m) {
        if (s != 0.f) {
            const float d = lse_ref(m) - lse_ref(mc), al = exp_of<true>(d);
            t = al * fmaf(s, d, t);
            s *= al;
        }
        m = mc;
    }
    const float r = lse_ref(m);
    float e[N], u[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
        e[i] = exp_of<true>(x[i] - r);
        u[i] = e[i] * fmaxf(x[i] - r, kF32Min);
    }
#pragma unroll
    for (int w = 1; w < N; w *= 2)
#pragma unroll
        for (int i = 0; i + w < N; i += 2 * w) e[i] += e[i + w], u[i] += u[i + w];
    s += e[0];
    t += u[0];
}

__device__ __forceinline__ void mst_merge(float& m, float& s, float& t, float m2, float s2, float t2) {
    if (m2 > m) {
        const float tm = m, ts = s, tt = t;
        m = m2; s = s2; t = t2; m2 = tm; s2 = ts; t2 = tt;
    }
    if (s2 != 0.f) {
        const float d = lse_ref(m2) - lse_ref(m), al = exp_of<true>(d);
        s += s2 * al;
        t += al * fmaf(s2, d, t2);
    }
}

// The per-token head of grpo.py / rloo.py.  In: lp_new, lp_old, lp_ref (GRPO only), the row's advantage, the clamp
// bounds fp32(1 - clip) / fp32(1 + clip), beta, and gt = d loss / d per_token_loss (the unit-upstream factor
// (1 / B) / sum_s(w) * w).  Out: the per-token loss, the clip indicator and d loss / d lp_new.  Gradients follow torch:
// min() splits a tie evenly between its two operands, clamp() passes the gradient at its edges.
struct TokenHead {
    float loss, clipped, dlp;
};

template <bool KL>
__device__ __forceinline__ TokenHead token_head(float lp_new, float lp_old, float lp_ref, float adv, float lo, float hi,
                                                float beta, float gt) {
    TokenHead h;
    const float ratio = expf(lp_new - lp_old);
    const float rc = ratio < lo ? lo : (ratio > hi ? hi : ratio);  // NaN stays NaN, as torch.clamp
    const float u = ratio * adv, c = rc * adv;
    float mn = u < c ? u : c;
    if (u != u) mn = u;  // torch.min propagates NaN from either side
    h.loss = -mn;
    const float gm = -gt;
    const float gu = u < c ? gm : (u == c ? 0.5f * gm : 0.f);
    const float gc = c < u ? gm : (u == c ? 0.5f * gm : 0.f);
    // clamp() passes its gradient by selection, as torch's where(): a NaN gt (a sequence whose weights sum to 0) reaches
    // only the rows whose selected branch carries it, so the NaN pattern is the reference's
    const bool inside = ratio >= lo && ratio <= hi;
    h.dlp = (gu * adv + (inside ? gc * adv : 0.f)) * ratio;
    if (KL) {
        const float dr = lp_ref - lp_new;
        const float e = expf(dr);
        h.loss = h.loss + beta * (e - dr - 1.f);
        const float gk = gt * beta;
        h.dlp -= gk * e - gk;
    }
    h.clipped = (ratio > hi || ratio < lo) ? 1.f : 0.f;
    return h;
}

// leave-one-out advantage of row b from reward (K, Bp): (k, j) = (b / Bp, b % Bp), baseline = (sum_k r[k, j] - r) / (K - 1),
// in fp64 and rounded once: rewards with a large common offset and a small spread cancel here, and an fp32 sum of K of
// them loses the spread (K equal rewards give exactly 0 only so)
__device__ __forceinline__ float rloo_adv(const float* __restrict__ reward, int K, long long Bp, long long b) {
    const long long k = b / Bp, j = b - k * Bp;
    double sum = 0.0;
    for (int q = 0; q < K; ++q) sum += (double)reward[(long long)q * Bp + j];
    const double r = reward[k * Bp + j];
    return (float)(r - (sum - r) / (double)(K - 1));
}

struct VocabArgs {
    const void* x[3];          // logit_new, logit_old, logit_ref (streams in that order; BWD / LOGP: x[0] only)
    const long long* action;   // (rows)
    const float* adv;          // GRPO: (B)
    const float* reward;       // RLOO: (K, B / K)
    const float* weight;       // (B, S) nullable = ones
    const float* coef_in;      // BWD: per-row coefficient
    const float* g;            // BWD: upstream scalar (nullable = 1)
    float* lp;                 // LOGP: (rows)
    float* lse;                // forward: logsumexp of logit_new per row; BWD: read
    float* coef;               // GRPO / RLOO: d loss / d lp_new per row for a unit upstream gradient
    void* grad;                // d / d logit_new (nullable in the forward = no gradient)
    float* ws;
    long long rows, S, V, Bp;
    int K, skip_if_unit, capv;  // capv: 16-byte vectors of logit_new kept in shared memory
    float lo, hi, beta, inv_b;
    // PPO (VM_PPO*, VM_PPO_BWD*); adv is then per row and coef / coef_in the policy term's unit coefficient
    float* ent;                // forward: entropy of logit_new per row (PPO_ENT); VM_PPO_BWD: read (null = no entropy)
    float* coef_kl;            // forward: d kl_div / d lp_new per row (PPO_KL); VM_PPO_BWD: read (null = no KL)
    UpstreamRecord rec;        // PPO forward and VM_PPO_BWD (slots policy, entropy, kl)
    float dual_clip, inv_m;    // dual_clip <= 0: off; inv_m = 1 / rows
    int kl_type;
    // A2C (VM_A2C, VM_PPO_BWD + PPO_ENT + PPO_VAL); adv is per row, rec also owns the value slot
    const float* value;        // forward: (rows)
    const float* ret;          // forward: return_ (rows)
    float* dval;               // forward: d value_loss / d value per row; backward: read
    float* grad_value;         // d / d value (rows), fp32
};

template <int NR, bool CACHE, class T, bool ENT = false>
__device__ __forceinline__ void stream_vecs(const uint4* const (&p)[NR], int i, float (&m)[NR], float (&s)[NR],
                                            uint4* cache, int capv, float* t = nullptr) {
    constexpr int W = VecT<T>::W;
    uint4 u[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) u[r] = r == 0 ? __ldg(p[0] + i) : __ldcs(p[r] + i);
    if (CACHE && i < capv) cache[i] = u[0];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        float x[W];
        VecT<T>::unpack(u[r], x);
        if (ENT && r == 0) mst_add<W>(m[0], s[0], *t, x);
        else ms_add<W, ENT>(m[r], s[r], x);
    }
}

template <class T, int MODE>
__global__ void __launch_bounds__(VOCAB_NT) vocab_rows_kernel(VocabArgs a) {
    pdl_prologue();
    using V_ = VecT<T>;
    constexpr int W = V_::W;
    constexpr bool PPO = MODE >= VM_PPO && MODE < VM_PPO_BWD, PBWD = MODE >= VM_PPO_BWD && MODE < VM_A2C;
    constexpr bool A2C = MODE == VM_A2C, VAL = A2C || (PBWD && (MODE & PPO_VAL));  // VAL: the A2C value slot
    constexpr bool ENT = ((PPO || PBWD) && (MODE & PPO_ENT)) || A2C, KL = PPO && (MODE & PPO_KL);
    constexpr bool BWD = MODE == VM_BWD || PBWD;
    constexpr int NR = MODE == VM_GRPO ? 3 : (MODE == VM_RLOO ? 2 : (PPO ? (KL ? 3 : 2) : 1));
    constexpr bool LOSS = MODE == VM_GRPO || MODE == VM_RLOO || PPO || A2C;
    constexpr int NP = PPO ? 5 : 3;
    extern __shared__ uint4 s_row[];
    __shared__ float s_m[NR][VOCAB_NT / 32], s_s[NR][VOCAB_NT / 32], s_w[VOCAB_NT / 32];
    __shared__ float s_c, s_lse;
    __shared__ long long s_a;
    __shared__ float s_t[ENT ? VOCAB_NT / 32 : 1], s_ce, s_h;  // PPO entropy: t partials, c_ent, H
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long V = a.V;
    const bool want_grad = a.grad != nullptr;
    float gscale = 1.f;
    if (MODE == VM_BWD) {
        if (a.g) gscale = *a.g;
        if (a.skip_if_unit && gscale == 1.f) return;  // the forward launch already wrote exactly this gradient
    }
    // PPO upstream-gradient slots: policy, entropy with the bonus, kl with logit_pretrained.  The record is written (forward)
    // or verified (VM_PPO_BWD) here; the values are read again where they are used, once per row, rather than held in
    // registers across the row loop.
    const unsigned owned = 1u | (VAL ? 2u : 0u) | (ENT ? 4u : 0u) | ((KL || (PBWD && a.coef_kl)) ? 8u : 0u);
    if (PBWD || ((PPO || A2C) && want_grad)) {
        float g[4];
        if (upstream<4>(a.rec, PBWD, owned, g)) return;  // VM_PPO_BWD: the forward wrote exactly this gradient
        if (PBWD && VAL) {
            // A2C: d / d value = g_val * dval, O(1) per row and always rewritten; d / d logit_new only when the policy
            // or entropy upstream gradient differs from the forward's (the gradient the forward wrote stays exact)
            for (long long r = (long long)blockIdx.x * VOCAB_NT + tid; r < a.rows; r += (long long)gridDim.x * VOCAB_NT)
                a.grad_value[r] = g[1] * a.dval[r];
            const float* u = a.rec.used;
            if (u && __float_as_uint(g[0]) == __float_as_uint(u[0]) && __float_as_uint(g[2]) == __float_as_uint(u[2]))
                return;
        }
    }
    float part[NP] = {0.f, 0.f, 0.f};  // thread 0: the loss partial sums of this CTA's rows (loss, approx_kl, clipfrac; PPO: 5)
    float w_tot = (float)a.S;  // thread 0: sum_s w[b, s] of the current row's sequence (S without weights)
    for (long long row = blockIdx.x; row < a.rows; row += gridDim.x) {
        const size_t off = (size_t)row * (size_t)V;
        // elements before the row's first 16-byte boundary (the base pointers are 16-byte aligned)
        const long long mis = (long long)((off * sizeof(T)) & 15u) / (long long)sizeof(T);
        const long long h = mis ? min((long long)(16 / sizeof(T)) - mis, V) : 0;
        const int nvec = (int)((V - h) / W);
        const long long tail0 = h + (long long)nvec * W;
        const T* rp[NR];
        const uint4* vp[NR];
#pragma unroll
        for (int r = 0; r < NR; ++r) {
            rp[r] = reinterpret_cast<const T*>(a.x[r]) + off;
            vp[r] = reinterpret_cast<const uint4*>(rp[r] + h);
        }
        float c = 0.f, lse = 0.f, ce = 0.f, H = 0.f;  // ce, H: PPO entropy term
        long long act = 0;
        if (MODE == VM_BWD) {
            c = gscale * a.coef_in[row];
            lse = a.lse[row];
            act = a.action[row];
        } else if (PBWD) {
            const float gp = upstream_value(a.rec, owned, 0), gk = upstream_value(a.rec, owned, 3);
            c = gp * a.coef_in[row] + (a.coef_kl ? gk * a.coef_kl[row] : 0.f);
            if (ENT) {
                ce = upstream_value(a.rec, owned, 2) * (a.weight ? a.weight[row] : 1.f) * a.inv_m;
                H = a.ent[row];
            }
            lse = a.lse[row];
            act = a.action[row];
        } else {
            float m[NR], s[NR], t = 0.f;  // t: PPO entropy accumulator of logit_new
#pragma unroll
            for (int r = 0; r < NR; ++r) m[r] = -INFINITY, s[r] = 0.f;
            const bool cache = LOSS && want_grad;
            int i = tid;
            for (; i + VOCAB_NT < nvec; i += 2 * VOCAB_NT) {
                if (cache) {
                    stream_vecs<NR, true, T, ENT>(vp, i, m, s, s_row, a.capv, &t);
                    stream_vecs<NR, true, T, ENT>(vp, i + VOCAB_NT, m, s, s_row, a.capv, &t);
                } else {
                    stream_vecs<NR, false, T, ENT>(vp, i, m, s, s_row, 0, &t);
                    stream_vecs<NR, false, T, ENT>(vp, i + VOCAB_NT, m, s, s_row, 0, &t);
                }
            }
            if (i < nvec) {
                if (cache) stream_vecs<NR, true, T, ENT>(vp, i, m, s, s_row, a.capv, &t);
                else stream_vecs<NR, false, T, ENT>(vp, i, m, s, s_row, 0, &t);
            }
            // the unaligned head and tail, < 16 bytes each
            for (long long j = tid; j < h + (V - tail0); j += VOCAB_NT) {
                const long long e = j < h ? j : tail0 + (j - h);
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    const float x[1] = {V_::to_f(rp[r][e])};
                    if (ENT && r == 0) mst_add<1>(m[0], s[0], t, x);
                    else ms_add<1, ENT>(m[r], s[r], x);
                }
            }
            float wsum = 0.f;
            // a CTA's rows step by gridDim.x (< S at language-model sizes): it sums a sequence's weights once per visit to
            // that sequence, not once per token
            const bool new_seq = (MODE == VM_GRPO || MODE == VM_RLOO) && a.weight &&
                                 (row < gridDim.x || row / a.S != (row - gridDim.x) / a.S);
            if (new_seq) {
                const float* wr = a.weight + (row / a.S) * a.S;
                for (long long j = tid; j < a.S; j += VOCAB_NT) wsum += wr[j];
            }
#pragma unroll
            for (int r = 0; r < NR; ++r) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float m2 = __shfl_down_sync(0xffffffffu, m[r], o), s2 = __shfl_down_sync(0xffffffffu, s[r], o);
                    if (ENT && r == 0) mst_merge(m[0], s[0], t, m2, s2, __shfl_down_sync(0xffffffffu, t, o));
                    else ms_merge<ENT>(m[r], s[r], m2, s2);
                }
                if (lane == 0) s_m[r][wid] = m[r], s_s[r][wid] = s[r];
            }
            if (ENT && lane == 0) s_t[wid] = t;
            if (new_seq) {
                wsum = warp_sum(wsum);
                if (lane == 0) s_w[wid] = wsum;
            }
            __syncthreads();
            if (tid == 0) {
                float lp[NR];
                act = a.action[row];
                const bool ok = act >= 0 && act < V;
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    float mm = s_m[r][0], ss = s_s[r][0];
                    if (ENT && r == 0) {
                        float tt = s_t[0];
                        for (int w = 1; w < VOCAB_NT / 32; ++w) mst_merge(mm, ss, tt, s_m[0][w], s_s[0][w], s_t[w]);
                        H = logf(ss) - tt / ss;
                    } else {
                        for (int w = 1; w < VOCAB_NT / 32; ++w) ms_merge<ENT>(mm, ss, s_m[r][w], s_s[r][w]);
                    }
                    const float l = logf(ss) + lse_ref(mm);
                    if (r == 0) lse = l;
                    lp[r] = ok ? V_::to_f(rp[r][act]) - l : __int_as_float(0x7fc00000);
                }
                a.lse[row] = lse;
                if (MODE == VM_LOGP) a.lp[row] = lp[0];
                if constexpr (PPO) {
                    const float w = a.weight ? a.weight[row] : 1.f;
                    const float ratio = expf(lp[0] - lp[1]);
                    float dsel, dk = 0.f, klv = 0.f;
                    const float adv = a.adv[row];
                    float sel = surrogate(ratio, adv, a.lo, a.hi, a.dual_clip, dsel);
                    if (ratio * adv != ratio * adv) sel = __int_as_float(0x7fc00000);  // torch.min / max propagate NaN
                    const float cp = -w * a.inv_m * dsel * ratio;  // d policy_loss / d lp_new
                    a.coef[row] = cp;
                    if (KL) {
                        klv = kl_term(lp[0] - lp[NR - 1], a.kl_type, dk);
                        a.coef_kl[row] = dk * a.inv_m;  // d kl_div / d lp_new
                    }
                    if (ENT) a.ent[row] = H;
                    if (want_grad) {
                        c = upstream_value(a.rec, owned, 0) * cp +
                            (KL ? upstream_value(a.rec, owned, 3) * dk * a.inv_m : 0.f);
                        ce = upstream_value(a.rec, owned, 2) * w * a.inv_m;
                    }
                    part[0] -= sel * w;
                    part[1] += H * w;
                    part[2] += klv;
                    part[3] += lp[1] - lp[0];
                    part[4] += (ratio > a.hi || ratio < a.lo) ? 1.f : 0.f;
                    s_ce = ce;
                    s_h = H;
                } else if constexpr (A2C) {  // a2c.py:39-44, in its operation order
                    const float w = a.weight ? a.weight[row] : 1.f;
                    const float adv = a.adv[row];
                    const float dv = a.ret[row] - a.value[row];
                    const float cp = -adv * w * a.inv_m;            // d policy_loss / d lp
                    const float dvu = -2.f * w * dv * a.inv_m;      // d value_loss / d value
                    a.coef[row] = cp;
                    a.dval[row] = dvu;
                    a.ent[row] = H;
                    if (want_grad) {
                        c = upstream_value(a.rec, owned, 0) * cp;
                        ce = upstream_value(a.rec, owned, 2) * w * a.inv_m;
                        a.grad_value[row] = upstream_value(a.rec, owned, 1) * dvu;
                    }
                    part[0] -= lp[0] * adv * w;
                    part[1] += dv * dv * w;
                    part[2] += H * w;
                    s_ce = ce;
                    s_h = H;
                } else if (LOSS) {
                    const long long b = row / a.S;
                    if (new_seq) {
                        w_tot = 0.f;
                        for (int w = 0; w < VOCAB_NT / 32; ++w) w_tot += s_w[w];
                    }
                    const float W_ = w_tot;
                    const float w = a.weight ? a.weight[row] : 1.f;
                    const float adv = MODE == VM_GRPO ? a.adv[b] : rloo_adv(a.reward, a.K, a.Bp, b);
                    const float gt = a.inv_b / W_ * w;
                    const TokenHead th = token_head<MODE == VM_GRPO>(lp[0], lp[1], NR > 2 ? lp[NR - 1] : 0.f, adv, a.lo,
                                                                     a.hi, a.beta, gt);
                    c = th.dlp;
                    a.coef[row] = c;
                    part[0] += th.loss * w / W_;
                    part[1] += lp[1] - lp[0];
                    part[2] += th.clipped;
                }
                s_c = c;
                s_lse = lse;
                s_a = act;
            }
            __syncthreads();
            if (!LOSS || !want_grad) continue;
            c = s_c;
            lse = s_lse;
            act = s_a;
            if (ENT) ce = s_ce, H = s_h;
        }
        // d / d logit_new[row] = c * (onehot(a) - softmax) [PPO entropy: - ce * p * (max(log p, -FLT_MAX) + H)]
        T* gr = reinterpret_cast<T*>(a.grad) + off;
        uint4* gv = reinterpret_cast<uint4*>(gr + h);
        for (int i = tid; i < nvec; i += VOCAB_NT) {
            const uint4 u = (LOSS && i < a.capv) ? s_row[i] : (BWD ? __ldcs(vp[0] + i) : __ldg(vp[0] + i));
            float x[W];
            V_::unpack(u, x);
            const long long e0 = h + (long long)i * W;
#pragma unroll
            for (int k = 0; k < W; ++k) {
                if (ENT) {
                    const float z = x[k] - lse, p = exp2f(z * kL2E);
                    x[k] = c * ((e0 + k == act ? 1.f : 0.f) - p) - ce * p * (fmaxf(z, kF32Min) + H);
                } else {
                    x[k] = c * ((e0 + k == act ? 1.f : 0.f) - exp2f((x[k] - lse) * kL2E));
                }
            }
            __stcs(gv + i, V_::pack(x));
        }
        for (long long j = tid; j < h + (V - tail0); j += VOCAB_NT) {
            const long long e = j < h ? j : tail0 + (j - h);
            const float x = V_::to_f(rp[0][e]);
            if (ENT) {
                const float z = x - lse, p = exp2f(z * kL2E);
                gr[e] = V_::from_f(c * ((e == act ? 1.f : 0.f) - p) - ce * p * (fmaxf(z, kF32Min) + H));
            } else {
                gr[e] = V_::from_f(c * ((e == act ? 1.f : 0.f) - exp2f((x - lse) * kL2E)));
            }
        }
        if (LOSS) __syncthreads();  // s_row and s_c are rewritten by the next row
    }
    if (LOSS) {
        float v[NP] = {0.f, 0.f, 0.f};
        if (tid == 0) v[0] = part[0], v[1] = part[1], v[2] = part[2];
        if constexpr (PPO) {
            if (tid == 0) v[3] = part[3], v[4] = part[4];
        }
        grid_store_partials<NP, VOCAB_NT>(v, a.ws);
    }
}

// The token head alone, on per-token log-probabilities a caller computed itself (a custom log_prob_fn): one CTA per
// sequence b at a time, thread = token.  Writes d loss / d lp_new for a unit upstream gradient and the loss partials.
template <bool KL>
__global__ void __launch_bounds__(VOCAB_HEAD_NT) token_head_kernel(const float* __restrict__ lp_new,
                                                                   const float* __restrict__ lp_old,
                                                                   const float* __restrict__ lp_ref, VocabArgs a) {
    pdl_prologue();
    __shared__ float s_w[VOCAB_HEAD_NT / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long B = a.rows / a.S;
    float part[3] = {0.f, 0.f, 0.f};
    for (long long b = blockIdx.x; b < B; b += gridDim.x) {
        const long long o = b * a.S;
        float W_ = (float)a.S;
        if (a.weight) {
            float ws = 0.f;
            for (long long j = tid; j < a.S; j += VOCAB_HEAD_NT) ws += a.weight[o + j];
            ws = warp_sum(ws);
            if (lane == 0) s_w[wid] = ws;
            __syncthreads();
            W_ = 0.f;
            for (int w = 0; w < VOCAB_HEAD_NT / 32; ++w) W_ += s_w[w];
            __syncthreads();
        }
        const float adv = KL ? a.adv[b] : rloo_adv(a.reward, a.K, a.Bp, b);
        for (long long j = tid; j < a.S; j += VOCAB_HEAD_NT) {
            const float w = a.weight ? a.weight[o + j] : 1.f;
            const float ln = lp_new[o + j], lo_ = lp_old[o + j];
            const TokenHead th = token_head<KL>(ln, lo_, KL ? lp_ref[o + j] : 0.f, adv, a.lo, a.hi, a.beta, a.inv_b / W_ * w);
            a.coef[o + j] = th.dlp;
            part[0] += th.loss * w / W_;
            part[1] += lo_ - ln;
            part[2] += th.clipped;
        }
    }
    grid_store_partials<3, VOCAB_HEAD_NT>(part, a.ws);
}

}  // namespace b200rl

using namespace b200rl;

namespace {

bool aligned_logits(const void* p) { return p && aligned16(p); }

template <class T, int MODE>
int launch_rows(VocabArgs& a, float* out3, size_t ws_bytes, long long B, cudaStream_t st) {
    constexpr auto kern = vocab_rows_kernel<T, MODE>;
    constexpr bool PPO = MODE >= VM_PPO && MODE < VM_PPO_BWD;
    constexpr bool LOSS = MODE == VM_GRPO || MODE == VM_RLOO || PPO || MODE == VM_A2C;
    constexpr int NP = PPO ? 5 : 3;
    const long long nvec_max = (a.V * (long long)sizeof(T) + 15) / 16;
    a.capv = (LOSS && a.grad) ? (int)min(nvec_max, (long long)(VOCAB_SMEM_CAP / 16)) : 0;
    const size_t smem = (size_t)a.capv * 16;
    int sms = 0, per_sm = 0;
    if (int rc = resident_ctas<kern>(VOCAB_NT, smem, sms, per_sm)) return rc;
    long long grid = (long long)sms * per_sm;
    if (grid > a.rows) grid = a.rows;
    if (LOSS && !ws_partials_fit(grid * NP, ws_bytes)) return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, VOCAB_NT, smem, st, a)) return rc;
    if (!LOSS) return B200RL_OK;
    FinalizeArgs fa{};
    if (PPO || MODE == VM_A2C) {  // PPO: policy, entropy, kl, approx_kl, clipfrac; A2C: policy, value, entropy; row means
        for (int k = 0; k < NP; ++k) fa.scale[k] = 1.0 / (double)a.rows;
    } else {
        fa.scale[0] = 1.0 / (double)B;
        fa.scale[1] = fa.scale[2] = 1.0 / (double)a.rows;
    }
    fa.k = NP;
    fa.n_blocks = (int)grid;
    return launch_finalize(a.ws, out3, fa, st);
}

template <int MODE>
int launch_dtype(int dtype, VocabArgs& a, float* out3, size_t ws_bytes, long long B, cudaStream_t st) {
    if (dtype == B200RL_DTYPE_F32) return launch_rows<float, MODE>(a, out3, ws_bytes, B, st);
    if (dtype == B200RL_DTYPE_BF16) return launch_rows<__nv_bfloat16, MODE>(a, out3, ws_bytes, B, st);
    return B200RL_ERR_ARG;
}

bool sizes_ok(long long B, long long S, long long V) {
    return B > 0 && S > 0 && V > 0 && V < (1ll << 31) && B * S < (1ll << 40);
}

}  // namespace

extern "C" int b200rl_grpo_fwd_grad(int dtype, const void* logit_new, const void* logit_old, const void* logit_ref,
                                    const long long* action, const float* adv, const float* weight, long long B,
                                    long long S, long long V, double clip_ratio, double beta, float* out3, float* lse_new,
                                    float* dlogp_unit, void* grad_logit_new, float* workspace, size_t workspace_bytes,
                                    void* stream) {
    if (!sizes_ok(B, S, V) || !aligned_logits(logit_new) || !aligned_logits(logit_old) || !aligned_logits(logit_ref) ||
        !action || !adv || !out3 || !lse_new || !dlogp_unit || !workspace ||
        (grad_logit_new && !aligned16(grad_logit_new)))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logit_new; a.x[1] = logit_old; a.x[2] = logit_ref;
    a.action = action; a.adv = adv; a.weight = weight;
    a.lse = lse_new; a.coef = dlogp_unit; a.grad = grad_logit_new; a.ws = workspace;
    a.rows = B * S; a.S = S; a.V = V;
    a.lo = (float)(1.0 - clip_ratio); a.hi = (float)(1.0 + clip_ratio); a.beta = (float)beta;
    a.inv_b = (float)(1.0 / (double)B);
    return launch_dtype<VM_GRPO>(dtype, a, out3, workspace_bytes, B, (cudaStream_t)stream);
}

extern "C" int b200rl_rloo_fwd_grad(int dtype, const void* logit_new, const void* logit_old, const long long* action,
                                    const float* reward, long long K, const float* weight, long long B, long long S,
                                    long long V, double clip_ratio, float* out3, float* lse_new, float* dlogp_unit,
                                    void* grad_logit_new, float* workspace, size_t workspace_bytes, void* stream) {
    if (!sizes_ok(B, S, V) || K < 1 || K > (1 << 20) || B % K || !aligned_logits(logit_new) ||
        !aligned_logits(logit_old) || !action || !reward || !out3 || !lse_new || !dlogp_unit || !workspace ||
        (grad_logit_new && !aligned16(grad_logit_new)))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logit_new; a.x[1] = logit_old;
    a.action = action; a.reward = reward; a.K = (int)K; a.Bp = B / K; a.weight = weight;
    a.lse = lse_new; a.coef = dlogp_unit; a.grad = grad_logit_new; a.ws = workspace;
    a.rows = B * S; a.S = S; a.V = V;
    a.lo = (float)(1.0 - clip_ratio); a.hi = (float)(1.0 + clip_ratio);
    a.inv_b = (float)(1.0 / (double)B);
    return launch_dtype<VM_RLOO>(dtype, a, out3, workspace_bytes, B, (cudaStream_t)stream);
}

extern "C" int b200rl_ppo_lm_fwd_grad(int dtype, const void* logit_new, const void* logit_old,
                                      const void* logit_pretrained, const long long* action, const float* adv,
                                      const float* weight, long long rows, long long V, double clip_ratio,
                                      double dual_clip, int kl_type, int entropy, const float* g_expected, float* g_used,
                                      float* out5, float* lse_new, float* entropy_row, float* dlogp_policy,
                                      float* dlogp_kl, void* grad_logit_new, float* workspace, size_t workspace_bytes,
                                      void* stream) {
    const bool kl = logit_pretrained != nullptr;
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logit_new) || !aligned_logits(logit_old) ||
        (kl && (!aligned16(logit_pretrained) || !dlogp_kl || kl_type < 1 || kl_type > 3)) || !action || !adv ||
        !lse_new || !dlogp_policy || (entropy && !entropy_row) || !workspace ||
        (grad_logit_new && !aligned16(grad_logit_new)) ||
        !upstream_args_ok(0, out5, grad_logit_new, grad_logit_new, g_expected, g_used))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logit_new; a.x[1] = logit_old; a.x[2] = logit_pretrained;
    a.action = action; a.adv = adv; a.weight = weight;
    a.lse = lse_new; a.coef = dlogp_policy; a.coef_kl = dlogp_kl; a.ent = entropy_row; a.grad = grad_logit_new;
    a.ws = workspace;
    a.rec = forward_record(g_expected, g_used);
    a.rows = rows; a.S = 1; a.V = V;
    a.lo = (float)(1.0 - clip_ratio); a.hi = (float)(1.0 + clip_ratio); a.dual_clip = (float)dual_clip;
    a.kl_type = kl_type; a.inv_m = (float)(1.0 / (double)rows);
    cudaStream_t st = (cudaStream_t)stream;
    const int mode = VM_PPO + (entropy ? PPO_ENT : 0) + (kl ? PPO_KL : 0);
    switch (mode) {
        case VM_PPO: return launch_dtype<VM_PPO>(dtype, a, out5, workspace_bytes, rows, st);
        case VM_PPO + PPO_ENT: return launch_dtype<VM_PPO + PPO_ENT>(dtype, a, out5, workspace_bytes, rows, st);
        case VM_PPO + PPO_KL: return launch_dtype<VM_PPO + PPO_KL>(dtype, a, out5, workspace_bytes, rows, st);
        default: return launch_dtype<VM_PPO + PPO_ENT + PPO_KL>(dtype, a, out5, workspace_bytes, rows, st);
    }
}

extern "C" int b200rl_ppo_lm_bwd(int dtype, const void* logit_new, const long long* action, const float* weight,
                                 long long rows, long long V, const float* lse_new, const float* entropy_row,
                                 const float* dlogp_policy, const float* dlogp_kl, const float* g_policy,
                                 const float* g_entropy, const float* g_kl, const float* g_used, float* g_hint,
                                 void* grad_logit_new, void* stream) {
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logit_new) || !action || !lse_new || !dlogp_policy ||
        !upstream_args_ok(1, nullptr, true, grad_logit_new, nullptr, g_used) || !aligned16(grad_logit_new))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logit_new; a.action = action; a.weight = weight;
    a.lse = const_cast<float*>(lse_new); a.ent = const_cast<float*>(entropy_row); a.coef_in = dlogp_policy;
    a.coef_kl = const_cast<float*>(dlogp_kl);
    a.rec = verify_record(g_policy, nullptr, g_entropy, g_kl, g_used, g_hint);
    a.grad = grad_logit_new;
    a.rows = rows; a.S = 1; a.V = V;
    a.inv_m = (float)(1.0 / (double)rows);
    cudaStream_t st = (cudaStream_t)stream;
    if (entropy_row) return launch_dtype<VM_PPO_BWD + PPO_ENT>(dtype, a, nullptr, 0, rows, st);
    return launch_dtype<VM_PPO_BWD>(dtype, a, nullptr, 0, rows, st);
}

extern "C" int b200rl_a2c_lm_fwd_grad(int dtype, const void* logit, const long long* action, const float* value,
                                      const float* adv, const float* return_, const float* weight, long long rows,
                                      long long V, const float* g_expected, float* g_used, float* out3, float* lse,
                                      float* entropy_row, float* dlogp_policy, float* dvalue, void* grad_logit,
                                      float* grad_value, float* workspace, size_t workspace_bytes, void* stream) {
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logit) || !action || !value || !adv || !return_ || !lse ||
        !entropy_row || !dlogp_policy || !dvalue || !workspace || (grad_logit && !aligned16(grad_logit)) ||
        (grad_value && !grad_logit) ||
        !upstream_args_ok(0, out3, grad_logit != nullptr, grad_logit && grad_value, g_expected, g_used))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logit;
    a.action = action; a.adv = adv; a.weight = weight; a.value = value; a.ret = return_;
    a.lse = lse; a.ent = entropy_row; a.coef = dlogp_policy; a.dval = dvalue;
    a.grad = grad_logit; a.grad_value = grad_value; a.ws = workspace;
    a.rec = forward_record(g_expected, g_used);
    a.rows = rows; a.S = 1; a.V = V;
    a.inv_m = (float)(1.0 / (double)rows);
    return launch_dtype<VM_A2C>(dtype, a, out3, workspace_bytes, rows, (cudaStream_t)stream);
}

extern "C" int b200rl_a2c_lm_bwd(int dtype, const void* logit, const long long* action, const float* weight,
                                 long long rows, long long V, const float* lse, const float* entropy_row,
                                 const float* dlogp_policy, const float* dvalue, const float* g_policy,
                                 const float* g_value, const float* g_entropy, const float* g_used, float* g_hint,
                                 void* grad_logit, float* grad_value, void* stream) {
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logit) || !action || !lse || !entropy_row || !dlogp_policy ||
        !dvalue || !upstream_args_ok(1, nullptr, true, grad_logit && grad_value, nullptr, g_used) ||
        !aligned16(grad_logit))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logit; a.action = action; a.weight = weight;
    a.lse = const_cast<float*>(lse); a.ent = const_cast<float*>(entropy_row); a.coef_in = dlogp_policy;
    a.dval = const_cast<float*>(dvalue);
    a.rec = verify_record(g_policy, g_value, g_entropy, nullptr, g_used, g_hint);
    a.grad = grad_logit; a.grad_value = grad_value;
    a.rows = rows; a.S = 1; a.V = V;
    a.inv_m = (float)(1.0 / (double)rows);
    return launch_dtype<VM_PPO_BWD + PPO_ENT + PPO_VAL>(dtype, a, nullptr, 0, rows, (cudaStream_t)stream);
}

extern "C" int b200rl_token_logp_fwd(int dtype, const void* logits, const long long* index, long long rows, long long V,
                                     float* logp, float* lse, void* stream) {
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logits) || !index || !logp || !lse) return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logits; a.action = index; a.lp = logp; a.lse = lse;
    a.rows = rows; a.S = 1; a.V = V;
    return launch_dtype<VM_LOGP>(dtype, a, nullptr, 0, rows, (cudaStream_t)stream);
}

extern "C" int b200rl_token_logp_bwd(int dtype, const void* logits, const long long* index, const float* lse,
                                     const float* dlogp, const float* g_scale, int skip_if_unit, long long rows,
                                     long long V, void* grad_logits, void* stream) {
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logits) || !index || !lse || !dlogp || !grad_logits ||
        !aligned16(grad_logits) || (skip_if_unit && !g_scale))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logits; a.action = index; a.lse = const_cast<float*>(lse); a.coef_in = dlogp; a.g = g_scale;
    a.skip_if_unit = skip_if_unit; a.grad = grad_logits;
    a.rows = rows; a.S = 1; a.V = V;
    return launch_dtype<VM_BWD>(dtype, a, nullptr, 0, rows, (cudaStream_t)stream);
}

extern "C" int b200rl_token_head_fwd(const float* logp_new, const float* logp_old, const float* logp_ref,
                                     const float* adv, const float* reward, long long K, const float* weight, long long B,
                                     long long S, double clip_ratio, double beta, float* out3, float* dlogp_unit,
                                     float* workspace, size_t workspace_bytes, void* stream) {
    const bool grpo = logp_ref != nullptr;
    if (!sizes_ok(B, S, 1) || !logp_new || !logp_old || !out3 || !dlogp_unit || !workspace ||
        (grpo ? !adv : (!reward || K < 1 || K > (1 << 20) || B % K)))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.adv = adv; a.reward = reward; a.K = (int)K; a.Bp = grpo ? 0 : B / K; a.weight = weight;
    a.coef = dlogp_unit; a.ws = workspace;
    a.rows = B * S; a.S = S; a.V = 1;
    a.lo = (float)(1.0 - clip_ratio); a.hi = (float)(1.0 + clip_ratio); a.beta = (float)beta;
    a.inv_b = (float)(1.0 / (double)B);
    auto kern = grpo ? token_head_kernel<true> : token_head_kernel<false>;
    int sms = 0, per_sm = 0;
    if (int rc = grpo ? resident_ctas<token_head_kernel<true>>(VOCAB_HEAD_NT, 0, sms, per_sm)
                      : resident_ctas<token_head_kernel<false>>(VOCAB_HEAD_NT, 0, sms, per_sm))
        return rc;
    long long grid = (long long)sms * per_sm;
    if (grid > B) grid = B;
    if (!ws_partials_fit(grid * 3, workspace_bytes)) return B200RL_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = launch_k(kern, (int)grid, VOCAB_HEAD_NT, 0, st, logp_new, logp_old, logp_ref, a)) return rc;
    FinalizeArgs fa{};
    fa.scale[0] = 1.0 / (double)B;
    fa.scale[1] = fa.scale[2] = 1.0 / (double)a.rows;
    fa.k = 3;
    fa.n_blocks = (int)grid;
    return launch_finalize(workspace, out3, fa, st);
}
