// Vocabulary-scale token losses of the language-model policy-gradient family, on fp32 or bf16 logits:
//   grpo_policy_error                 ding/rl_utils/grpo.py             clipped ratio loss + beta * k3 KL to the reference policy
//   rloo_policy_error                 ding/rl_utils/rloo.py             clipped ratio loss, leave-one-out advantage from reward (K, B')
//   naive / efficient / less_efficient_method   ding/rl_utils/log_prob_utils.py   per-token log p(a) and its backward
//   ppo_policy_error / ppo_error's policy part  ding/rl_utils/ppo.py:143-230      on token rows (B, S, V)
//   a2c_error                                   ding/rl_utils/a2c.py:10-44        on token rows, with a per-token value head
// and the same losses from the lm_head's hidden states (rl_utils/lm_linear.py), one chunk of logits at a time.
//
// THE CORE, vocab_rows_kernel<T, Head>: persistent CTAs of VOCAB_NT threads, each owning one token row of V logits at a
// time (row += gridDim.x).  Per row, in ONE streaming pass over the head's Head::NR logit streams (16-byte vector loads,
// all streams' loads of an iteration in flight together), an online max / sum of exp in fp32 per stream gives
// logsumexp = max + log(sum exp(z - max)) with torch's rule for an infinite max (treated as 0); the gathered z[a] gives
// lp = z[a] - logsumexp.  With Head::ENT the pass also keeps, next to logit_new's max / sum,
// t = sum e^(z - r) * max(z - r, -FLT_MAX) (r the running max, rescaled with it like s), so H = log s - t / s reuses the
// exponentials already taken.  After the warp / CTA merge, thread 0 runs the head's row function on lp[] and H: it writes
// the head's per-row outputs, adds to the CTA's loss partials and returns (c, ce); the CTA then writes
//   d loss / d logit_new[row] = c * (onehot(a) - p) - ce * p * (max(log p, -FLT_MAX) + H),   p = softmax(logit_new[row])
// in T (ce = 0 without entropy).  A head that does not stream (the two backward heads) takes c, ce and H from the rows a
// forward launch saved and goes straight to that gradient pass.  Loss sums: per-CTA partials (grid_store_partials) added
// in a fixed order by finalize_sums_kernel -- deterministic, no atomics, no host sync.  One launch plan (launch_rows)
// serves whole tensors and chunks alike; a whole tensor is the one-chunk case.
//
// Traffic floor per token row: every logit stream read once plus the gradient written once, (NR + 1) * V * sizeof(T):
// (3 + 1) for GRPO and for PPO with logit_pretrained, (2 + 1) for RLOO and for PPO without, (1 + 1) for A2C and for every
// head on a chunk.  Per-row side data (action, weight, lse, coefficients, per-token operands) is O(1) per row.
//
// The softmax of the gradient needs logit_new a second time.  The streaming pass keeps the row in dynamic shared memory
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
// In place on a chunk (Head::INPL): from hidden states the caller computes the logits one chunk of token rows at a time
// into a (rows_per_chunk, V) buffer Z with a GEMM, and the chunk heads write d loss / d Z over Z itself, which the caller
// then feeds to the dH / dW GEMMs.  That is safe because (1) one CTA owns a row, (2) H and lse are known before the
// gradient pass because the streaming pass forms them, (3) each element's gradient is stored by the thread that has
// just read that element in the softmax pass (from the shared-memory copy, or from Z for the part past VOCAB_SMEM_CAP),
// and (4) nothing reads the row after that pass.  The logits and the gradient therefore alias: neither pointer is
// __restrict__ (VocabArgs holds plain pointers), and Z is read with coherent loads (__ldca), never the read-only path
// (__ldg), which requires the data to stay unwritten for the kernel's lifetime.  LogpRow and CoefBwdRow (whose
// load / store pair is already per element and coherent) run on chunk pointers unchanged.  Each chunk launches the same
// grid and its CTAs store their partials into the chunk's own slice of the workspace; the last chunk's launch adds all
// of them in one finalize_sums (a fixed chunk plan gives the same bits on every run).
//
// Forward-written gradients (the upstream-gradient record of common.cuh).  On logits, the PPO and A2C forward launches
// write d / d logit_new (and A2C's d / d value) for the upstream gradients the call site expects, read from the device
// and recorded as used, and save per row what a recompute needs: lse, H and the unit coefficients.  Their backward
// launch (PgBwdRow) verifies the record on the device: it returns at once when every owned upstream gradient is the one
// the forward used, and otherwise re-reads logit_new once and writes the gradient once from the saved rows.  GRPO / RLOO
// save the unit coefficient d loss / d lp_new, and CoefBwdRow applies the actual upstream scalar, returning at once
// when it is 1.  The chunk heads keep no record: the gradient of the one differentiable output, the loss mix, is fixed
// at launch, and the caller scales d Z's products dH / dW by its actual upstream gradient, which a per-component mix
// could not be once the chunk is gone.
//
// THE HEADS (each below, with its operands):
//   GrpoRow<KL, LIN>     GRPO (KL) / RLOO via token_head, in the reference's operation order.  On logits it streams
//                        logit_new, logit_old (and logit_ref) and sums a sequence's weights inside the row reduction, once
//                        per visit of a CTA to the sequence; on a chunk it reads per-token fp32 logp_old / logp_ref, and
//                        the sequence normalisers that couple rows across chunk boundaries (a chunk may split a
//                        sequence) come from lm_seq_kernel, launched once before the first chunk.
//   LogpRow              per-token log p(a) and lse (the log-prob methods, token_logp_linear).
//   CoefBwdRow           d / d logit_new from g * coef[row] (their backward; GRPO / RLOO's for a non-unit upstream).
//   PpoRow<ENT, KL, LIN> surrogate / kl_term of ppo_math.cuh via ppo_head, so a call carries only the streams and terms
//                        it has (the common RLHF call: no entropy, 2 or 3 streams).  Loss sums: policy, entropy, kl,
//                        approx_kl, clipfrac, all over M rows.  Upstream gradients: (g_pol, g_ent, g_kl) from the record
//                        on logits, the loss mix (1, w_ent, w_kl) on a chunk.
//   A2cRow<LIN>          a2c_head: lp, H, dv = return_ - value, partials -lp * adv * w, dv^2 * w, H * w, means over M;
//                        d / d value = g_val * (-2 * w * dv / M) in fp32, so the value head needs no second launch.
//   PgBwdRow<ENT, VAL>   the backward of PpoRow / A2cRow on logits; with A2C's value slot (VAL) it always rewrites
//                        d / d value (O(1) per row), and d / d logit_new only when g_pol or g_ent differs.
//
// The loss head on a custom log_prob_fn's (B, S) output is a second, small kernel (token_head_kernel below): it reads no
// logits, so it shares the head arithmetic (token_head) but none of the row machinery.
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200rl.h"
#include "common.cuh"
#include "ppo_math.cuh"

namespace b200rl {

constexpr int VOCAB_NT = 512;
constexpr int VOCAB_HEAD_NT = 256;
constexpr int VOCAB_SMEM_CAP = 220 * 1024;  // dynamic shared memory for the cached part of logit_new (227 KB opt-in max)
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
    const void* x[3];          // the head's logit streams: logit_new, logit_old, logit_ref / logit_pretrained
    const long long* action;   // (rows)
    const float* adv;          // GRPO: (B)
    const float* reward;       // RLOO: (K, B / K)
    const float* weight;       // (B, S) nullable = ones
    const float* coef_in;      // backward: per-row coefficient
    const float* g;            // CoefBwdRow: upstream scalar (nullable = 1)
    float* lp;                 // LogpRow, GrpoRow on a chunk (nullable): log p(a) (rows)
    float* lse;                // forward: logsumexp of logit_new per row; backward: read
    float* coef;               // GRPO / RLOO: d loss / d lp_new per row for a unit upstream gradient
    void* grad;                // d / d logit_new (nullable in the forward = no gradient)
    float* ws;
    long long rows, S, V, Bp;
    int K, skip_if_unit, capv;  // capv: 16-byte vectors of logit_new kept in shared memory
    float lo, hi, beta, inv_b;
    // PpoRow, PgBwdRow; adv is then per row and coef / coef_in the policy term's unit coefficient
    float* ent;                // forward: entropy of logit_new per row (ENT); backward: read (null = no entropy)
    float* coef_kl;            // forward: d kl_div / d lp_new per row (KL); backward: read (null = no KL)
    UpstreamRecord rec;        // PpoRow / A2cRow on logits and PgBwdRow (slots policy, value, entropy, kl)
    float dual_clip, inv_m;    // dual_clip <= 0: off; inv_m = 1 / rows
    int kl_type;
    // A2cRow, PgBwdRow with the value slot; adv is per row
    const float* value;        // forward: (rows)
    const float* ret;          // forward: return_ (rows)
    float* dval;               // forward: d value_loss / d value per row; backward: read
    float* grad_value;         // d / d value (rows), fp32
    // GrpoRow on a chunk: the per-row operands start at the chunk's first row; the sequence index is (row0 + r) / S
    const float* lp_old;       // (rows)
    const float* lp_ref;       // GRPO: (rows)
    const float* seq;          // (2, nb): sum_s w[b, s], then the advantage of sequence b (lm_seq_kernel)
    long long row0, nb;        // nb: the number of sequences B (GrpoRow)
    // PpoRow / A2cRow on a chunk: the loss mix, i.e. the fixed upstream gradients of the entropy, kl and value terms (lp_ref
    // is then logp_pretrained; adv, value, ret and grad_value start at the chunk's first row)
    float w_ent, w_kl, w_val;
};

// The per-token PPO head of PpoRow (ppo.py:186-230, in its operation order): adds the five loss partials
// (policy, entropy, kl, approx_kl, clipfrac) to part and returns the unit coefficients d policy_loss / d lp_new and
// d kl_term / d lp_new (before the 1 / M of the mean)
struct PPOHead {
    float cp, dk;
};

template <bool KL>
__device__ __forceinline__ PPOHead ppo_head(const VocabArgs& a, float lp_new, float lp_old, float lp_pre, float adv,
                                            float w, float H, float* part) {
    PPOHead h;
    const float ratio = expf(lp_new - lp_old);
    float dsel, klv = 0.f;
    h.dk = 0.f;
    float sel = surrogate(ratio, adv, a.lo, a.hi, a.dual_clip, dsel);
    if (ratio * adv != ratio * adv) sel = __int_as_float(0x7fc00000);  // torch.min / max propagate NaN
    h.cp = -w * a.inv_m * dsel * ratio;  // d policy_loss / d lp_new
    if (KL) klv = kl_term(lp_new - lp_pre, a.kl_type, h.dk);
    part[0] -= sel * w;
    part[1] += H * w;
    part[2] += klv;
    part[3] += lp_old - lp_new;
    part[4] += (ratio > a.hi || ratio < a.lo) ? 1.f : 0.f;
    return h;
}

// The per-token A2C head of A2cRow (a2c.py:39-44, in its operation order): adds the three loss partials
// (policy, value, entropy) to part and returns d policy_loss / d lp and d value_loss / d value
struct A2CHead {
    float cp, dvu;
};

__device__ __forceinline__ A2CHead a2c_head(const VocabArgs& a, float lp, float adv, float ret, float value, float w,
                                            float H, float* part) {
    A2CHead h;
    const float dv = ret - value;
    h.cp = -adv * w * a.inv_m;
    h.dvu = -2.f * w * dv * a.inv_m;
    part[0] -= lp * adv * w;
    part[1] += dv * dv * w;
    part[2] += H * w;
    return h;
}

// INPL: stream 0 is the buffer the kernel overwrites with its gradient -- coherent loads, not the read-only path
template <int NR, bool CACHE, class T, bool ENT = false, bool INPL = false>
__device__ __forceinline__ void stream_vecs(const uint4* const (&p)[NR], int i, float (&m)[NR], float (&s)[NR],
                                            uint4* cache, int capv, float* t = nullptr) {
    constexpr int W = VecT<T>::W;
    uint4 u[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) u[r] = r == 0 ? (INPL ? __ldca(p[0] + i) : __ldg(p[0] + i)) : __ldcs(p[r] + i);
    if (CACHE && i < capv) cache[i] = u[0];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        float x[W];
        VecT<T>::unpack(u[r], x);
        if (ENT && r == 0) mst_add<W>(m[0], s[0], *t, x);
        else ms_add<W, ENT>(m[r], s[r], x);
    }
}

// d loss / d logit_new[row] = c * (onehot(a) - p) - ce * p * (max(log p, -FLT_MAX) + H): the coefficients a head returns
struct RowCoef {
    float c, ce;
};

// What the core knows of a launch before its row loop and hands to every head call: whether it writes a gradient, the
// upstream-record slots the head owns (common.cuh; 0 without a record) and CoefBwdRow's upstream scalar
struct RowLaunch {
    bool want_grad;
    unsigned owned;
    float g;
};

// What a head does not say: one stream, no loss sums, no entropy accumulator, the read-only path, streams the row, no
// sequence weight in the row reduction, every loss sum over the N rows of the call, no record, no prologue
struct HeadBase {
    static constexpr int NR = 1, NP = 0;
    static constexpr bool ENT = false, INPL = false, STREAM = true, SEQW = false, LOSS_OVER_B = false;
    static __device__ __forceinline__ unsigned owned(const VocabArgs&) { return 0u; }
    static __device__ __forceinline__ bool prologue(const VocabArgs&, RowLaunch&) { return false; }
};

// A forward head with a record on logits (not LIN): it owns the slots OWNED, and its prologue writes the values it applies
template <bool LIN, unsigned OWNED>
struct RecordHead : HeadBase {
    static __device__ __forceinline__ unsigned owned(const VocabArgs&) { return OWNED; }
    static __device__ __forceinline__ bool prologue(const VocabArgs& a, RowLaunch& L) {
        float g[4];
        if (!LIN && L.want_grad) upstream<4>(a.rec, false, L.owned, g);
        return false;
    }
};

// GRPO (KL) / RLOO; w_seq: the sequence's weight sum from the row reduction (logits).  Sums: loss, approx_kl, clipfrac
template <bool KL, bool LIN>
struct GrpoRow : HeadBase {
    static constexpr int NR = LIN ? 1 : (KL ? 3 : 2), NP = 3;
    static constexpr bool INPL = LIN, SEQW = !LIN, LOSS_OVER_B = true;
    static __device__ __forceinline__ RowCoef row(const VocabArgs& a, const RowLaunch&, long long row, const float* lp,
                                                  float lse, float, float w_seq, float* part) {
        a.lse[row] = lse;
        const long long b = LIN ? (a.row0 + row) / a.S : row / a.S;
        const float W_ = LIN ? a.seq[b] : w_seq;
        const float w = a.weight ? a.weight[row] : 1.f;
        const float adv = LIN ? a.seq[a.nb + b] : (KL ? a.adv[b] : rloo_adv(a.reward, a.K, a.Bp, b));
        const float lpo = LIN ? a.lp_old[row] : lp[1];
        const TokenHead th = token_head<KL>(lp[0], lpo, KL ? (LIN ? a.lp_ref[row] : lp[NR - 1]) : 0.f, adv, a.lo, a.hi,
                                            a.beta, a.inv_b / W_ * w);
        if (LIN && a.lp) a.lp[row] = lp[0];
        if (!LIN) a.coef[row] = th.dlp;
        part[0] += th.loss * w / W_;
        part[1] += lpo - lp[0];
        part[2] += th.clipped;
        return {th.dlp, 0.f};
    }
};

// log p(a) and logsumexp per row, no gradient
struct LogpRow : HeadBase {
    static __device__ __forceinline__ RowCoef row(const VocabArgs& a, const RowLaunch&, long long row, const float* lp,
                                                  float lse, float, float, float*) {
        a.lse[row] = lse;
        a.lp[row] = lp[0];
        return {0.f, 0.f};
    }
};

// c = g * coef[row] on the saved lse; with skip_if_unit it returns at once when g == 1 (the forward wrote this gradient)
struct CoefBwdRow : HeadBase {
    static constexpr bool STREAM = false;
    static __device__ __forceinline__ bool prologue(const VocabArgs& a, RowLaunch& L) {
        if (a.g) L.g = *a.g;
        return a.skip_if_unit && L.g == 1.f;
    }
    static __device__ __forceinline__ RowCoef coef(const VocabArgs& a, const RowLaunch& L, long long row, float&) {
        return {L.g * a.coef_in[row], 0.f};
    }
};

// PPO (ENT: entropy bonus, KL: pretrained log p given); upstream gradients: the record, or on a chunk (1, w_ent, w_kl)
template <bool ENT_, bool KL, bool LIN>
struct PpoRow : RecordHead<LIN, 1u | (ENT_ ? 4u : 0u) | (KL ? 8u : 0u)> {  // slots policy, entropy, kl
    static constexpr int NR = LIN ? 1 : (KL ? 3 : 2), NP = 5;
    static constexpr bool ENT = ENT_, INPL = LIN;
    static __device__ __forceinline__ RowCoef row(const VocabArgs& a, const RowLaunch& L, long long row, const float* lp,
                                                  float lse, float H, float, float* part) {
        if (!LIN) a.lse[row] = lse;
        const float w = a.weight ? a.weight[row] : 1.f;
        const PPOHead ph = ppo_head<KL>(a, lp[0], LIN ? a.lp_old[row] : lp[1],
                                        LIN ? (KL ? a.lp_ref[row] : 0.f) : lp[NR - 1], a.adv[row], w, H, part);
        if (!LIN) {
            a.coef[row] = ph.cp;
            if (KL) a.coef_kl[row] = ph.dk * a.inv_m;  // d kl_div / d lp_new
            if (ENT) a.ent[row] = H;
        }
        RowCoef r{0.f, 0.f};
        // The record is read here, once per row, rather than held across the row loop; each value is read where it is
        // used, as loading all first lets nvcc contract the other product of c into the FMA (a different last bit)
        if (LIN || L.want_grad) {
            r.c = (LIN ? 1.f : upstream_value(a.rec, L.owned, 0)) * ph.cp +
                  (KL ? (LIN ? a.w_kl : upstream_value(a.rec, L.owned, 3)) * ph.dk * a.inv_m : 0.f);
            r.ce = (LIN ? a.w_ent : upstream_value(a.rec, L.owned, 2)) * w * a.inv_m;
        }
        return r;
    }
};

// A2C; upstream gradients: the record, or on a chunk (1, w_val, w_ent), where d / d value is written only when wanted
template <bool LIN>
struct A2cRow : RecordHead<LIN, 7u> {  // slots policy, value, entropy
    static constexpr int NP = 3;
    static constexpr bool ENT = true, INPL = LIN;
    static __device__ __forceinline__ RowCoef row(const VocabArgs& a, const RowLaunch& L, long long row, const float* lp,
                                                  float lse, float H, float, float* part) {
        if (!LIN) a.lse[row] = lse;
        const float w = a.weight ? a.weight[row] : 1.f;
        const A2CHead ah = a2c_head(a, lp[0], a.adv[row], a.ret[row], a.value[row], w, H, part);
        if (!LIN) {
            a.coef[row] = ah.cp;
            a.dval[row] = ah.dvu;
            a.ent[row] = H;
        }
        RowCoef r{0.f, 0.f};
        if (LIN || L.want_grad) {
            const float gp = LIN ? 1.f : upstream_value(a.rec, L.owned, 0);
            const float gv = LIN ? a.w_val : upstream_value(a.rec, L.owned, 1);
            const float ge = LIN ? a.w_ent : upstream_value(a.rec, L.owned, 2);
            r.c = gp * ah.cp;
            r.ce = ge * w * a.inv_m;
            if (!LIN || a.grad_value) a.grad_value[row] = gv * ah.dvu;
        }
        return r;
    }
};

// The verify launch of PpoRow / A2cRow on logits (ENT: entropy saved, VAL: A2C's value slot, kl when coef_kl is given)
template <bool ENT_, bool VAL>
struct PgBwdRow : HeadBase {
    static constexpr bool ENT = ENT_, STREAM = false;
    static __device__ __forceinline__ unsigned owned(const VocabArgs& a) {
        return 1u | (VAL ? 2u : 0u) | (ENT ? 4u : 0u) | (a.coef_kl ? 8u : 0u);
    }
    static __device__ __forceinline__ bool prologue(const VocabArgs& a, RowLaunch& L) {
        float g[4];
        if (upstream<4>(a.rec, true, L.owned, g)) return true;
        if (VAL) {
            for (long long r = (long long)blockIdx.x * VOCAB_NT + threadIdx.x; r < a.rows;
                 r += (long long)gridDim.x * VOCAB_NT)
                a.grad_value[r] = g[1] * a.dval[r];
            const float* u = a.rec.used;
            if (u && __float_as_uint(g[0]) == __float_as_uint(u[0]) && __float_as_uint(g[2]) == __float_as_uint(u[2]))
                return true;
        }
        return false;
    }
    static __device__ __forceinline__ RowCoef coef(const VocabArgs& a, const RowLaunch& L, long long row, float& H) {
        const float gp = upstream_value(a.rec, L.owned, 0), gk = upstream_value(a.rec, L.owned, 3);
        RowCoef r{gp * a.coef_in[row] + (a.coef_kl ? gk * a.coef_kl[row] : 0.f), 0.f};
        if (ENT) {
            r.ce = upstream_value(a.rec, L.owned, 2) * (a.weight ? a.weight[row] : 1.f) * a.inv_m;
            H = a.ent[row];
        }
        return r;
    }
};

template <class T, class Head>
__global__ void __launch_bounds__(VOCAB_NT) vocab_rows_kernel(VocabArgs a) {
    pdl_prologue();
    using V_ = VecT<T>;
    constexpr int W = V_::W, NR = Head::NR, NP = Head::NP;
    constexpr bool ENT = Head::ENT, INPL = Head::INPL, STREAM = Head::STREAM, LOSS = NP > 0;
    extern __shared__ uint4 s_row[];
    __shared__ float s_m[NR][VOCAB_NT / 32], s_s[NR][VOCAB_NT / 32], s_w[VOCAB_NT / 32];
    __shared__ float s_c, s_lse;
    __shared__ long long s_a;
    __shared__ float s_t[ENT ? VOCAB_NT / 32 : 1], s_ce, s_h;  // entropy: t partials, c_ent, H
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long V = a.V;
    RowLaunch L{a.grad != nullptr, Head::owned(a), 1.f};
    if (Head::prologue(a, L)) return;
    float part[LOSS ? NP : 1] = {};  // thread 0: the loss partial sums of this CTA's rows
    float w_tot = (float)a.S;  // thread 0: sum_s w[b, s] of the current row's sequence (SEQW; S without weights)
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
        float c = 0.f, lse = 0.f, ce = 0.f, H = 0.f;  // ce, H: entropy term
        long long act = 0;
        if constexpr (!STREAM) {
            const RowCoef rc = Head::coef(a, L, row, H);
            c = rc.c;
            ce = rc.ce;
            lse = a.lse[row];
            act = a.action[row];
        } else {
            float m[NR], s[NR], t = 0.f;  // t: entropy accumulator of logit_new
#pragma unroll
            for (int r = 0; r < NR; ++r) m[r] = -INFINITY, s[r] = 0.f;
            const bool cache = LOSS && L.want_grad;
            int i = tid;
            for (; i + VOCAB_NT < nvec; i += 2 * VOCAB_NT) {
                if (cache) {
                    stream_vecs<NR, true, T, ENT, INPL>(vp, i, m, s, s_row, a.capv, &t);
                    stream_vecs<NR, true, T, ENT, INPL>(vp, i + VOCAB_NT, m, s, s_row, a.capv, &t);
                } else {
                    stream_vecs<NR, false, T, ENT, INPL>(vp, i, m, s, s_row, 0, &t);
                    stream_vecs<NR, false, T, ENT, INPL>(vp, i + VOCAB_NT, m, s, s_row, 0, &t);
                }
            }
            if (i < nvec) {
                if (cache) stream_vecs<NR, true, T, ENT, INPL>(vp, i, m, s, s_row, a.capv, &t);
                else stream_vecs<NR, false, T, ENT, INPL>(vp, i, m, s, s_row, 0, &t);
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
            // that sequence, not once per token, here in the row reduction so that it shares the reduction's barrier
            const bool new_seq = Head::SEQW && a.weight && (row < gridDim.x || row / a.S != (row - gridDim.x) / a.S);
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
                if (new_seq) {
                    w_tot = 0.f;
                    for (int w = 0; w < VOCAB_NT / 32; ++w) w_tot += s_w[w];
                }
                const RowCoef rc = Head::row(a, L, row, lp, lse, H, w_tot, part);
                s_c = rc.c;
                s_lse = lse;
                s_a = act;
                if (ENT) s_ce = rc.ce, s_h = H;
            }
            __syncthreads();
            if (!LOSS || !L.want_grad) continue;
            c = s_c;
            lse = s_lse;
            act = s_a;
            if (ENT) ce = s_ce, H = s_h;
        }
        // d / d logit_new[row] = c * (onehot(a) - softmax) [entropy: - ce * p * (max(log p, -FLT_MAX) + H)]
        T* gr = reinterpret_cast<T*>(a.grad) + off;
        uint4* gv = reinterpret_cast<uint4*>(gr + h);
        for (int i = tid; i < nvec; i += VOCAB_NT) {
            const uint4 u = (STREAM && i < a.capv) ? s_row[i]
                                                   : (!STREAM ? __ldcs(vp[0] + i) : (INPL ? __ldca(vp[0] + i) : __ldg(vp[0] + i)));
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
    if constexpr (LOSS) {
        float v[NP] = {};
        if (tid == 0)
#pragma unroll
            for (int k = 0; k < NP; ++k) v[k] = part[k];
        grid_store_partials<NP, VOCAB_NT>(v, a.ws);
    }
}

// sum_s w[b, s] of the sequence whose S weights start at weight + o (S without weights), in every thread of a
// VOCAB_HEAD_NT-thread CTA
__device__ __forceinline__ float seq_weight_sum(const float* weight, long long o, long long S) {
    __shared__ float s_w[VOCAB_HEAD_NT / 32];
    if (!weight) return (float)S;
    const int tid = threadIdx.x;
    float ws = 0.f;
    for (long long j = tid; j < S; j += VOCAB_HEAD_NT) ws += weight[o + j];
    ws = warp_sum(ws);
    if ((tid & 31) == 0) s_w[tid >> 5] = ws;
    __syncthreads();
    float W_ = 0.f;
    for (int w = 0; w < VOCAB_HEAD_NT / 32; ++w) W_ += s_w[w];
    __syncthreads();
    return W_;
}

// The token head alone, on per-token log-probabilities a caller computed itself (a custom log_prob_fn): one CTA per
// sequence b at a time, thread = token.  Writes d loss / d lp_new for a unit upstream gradient and the loss partials.
template <bool KL>
__global__ void __launch_bounds__(VOCAB_HEAD_NT) token_head_kernel(const float* __restrict__ lp_new,
                                                                   const float* __restrict__ lp_old,
                                                                   const float* __restrict__ lp_ref, VocabArgs a) {
    pdl_prologue();
    const int tid = threadIdx.x;
    const long long B = a.rows / a.S;
    float part[3] = {0.f, 0.f, 0.f};
    for (long long b = blockIdx.x; b < B; b += gridDim.x) {
        const long long o = b * a.S;
        const float W_ = seq_weight_sum(a.weight, o, a.S);
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

// The sequence normalisers of GrpoRow on a chunk, once per call: one CTA per sequence b at a time writes
// seq[b] = sum_s w[b, s] (token_head_kernel's sum) and seq[nb + b] = the advantage of sequence b.
__global__ void __launch_bounds__(VOCAB_HEAD_NT) lm_seq_kernel(VocabArgs a) {
    pdl_prologue();
    float* seq = const_cast<float*>(a.seq);
    for (long long b = blockIdx.x; b < a.nb; b += gridDim.x) {
        const float W_ = seq_weight_sum(a.weight, b * a.S, a.S);
        if (threadIdx.x == 0) {
            seq[b] = W_;
            seq[a.nb + b] = a.reward ? rloo_adv(a.reward, a.K, a.Bp, b) : a.adv[b];
        }
    }
}

// x *= *g in place, in T, skipped on the device when *g == 1: the backward of the hidden-state losses scales the dH / dW
// their forward wrote for a unit upstream gradient (b200rl_scale is fp32-only and out of place, which would hold a second
// copy of a 2 GB dW)
template <class T>
__global__ void __launch_bounds__(256) scale_inplace_kernel(const float* __restrict__ g, T* x, long long n) {
    pdl_prologue();
    using V_ = VecT<T>;
    constexpr int W = V_::W;
    const float s = *g;
    if (s == 1.f) return;
    const long long nv = n / W, step = (long long)gridDim.x * blockDim.x;
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    uint4* xv = reinterpret_cast<uint4*>(x);
    for (long long i = t0; i < nv; i += step) {
        float v[W];
        V_::unpack(xv[i], v);
#pragma unroll
        for (int k = 0; k < W; ++k) v[k] = s * v[k];
        xv[i] = V_::pack(v);
    }
    for (long long i = nv * W + t0; i < n; i += step) x[i] = V_::from_f(s * V_::to_f(x[i]));
}

// out = *g * in, in T, always written: the out-of-place form of scale_inplace_kernel for a backward that may not hand
// back the buffer its forward wrote (a torch.library op).  Same bits: s * v rounded to T, and in's bits when *g == 1.
template <class T>
__global__ void __launch_bounds__(256) scale_out_kernel(const float* __restrict__ g, const T* __restrict__ in,
                                                        T* __restrict__ out, long long n) {
    pdl_prologue();
    using V_ = VecT<T>;
    constexpr int W = V_::W;
    const float s = *g;
    const long long nv = n / W, step = (long long)gridDim.x * blockDim.x;
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const uint4* iv = reinterpret_cast<const uint4*>(in);
    uint4* ov = reinterpret_cast<uint4*>(out);
    if (s == 1.f) {
        for (long long i = t0; i < nv; i += step) ov[i] = iv[i];
        for (long long i = nv * W + t0; i < n; i += step) out[i] = in[i];
        return;
    }
    for (long long i = t0; i < nv; i += step) {
        float v[W];
        V_::unpack(iv[i], v);
#pragma unroll
        for (int k = 0; k < W; ++k) v[k] = s * v[k];
        ov[i] = V_::pack(v);
    }
    for (long long i = nv * W + t0; i < n; i += step) out[i] = V_::from_f(s * V_::to_f(in[i]));
}

}  // namespace b200rl

using namespace b200rl;

namespace {

bool aligned_logits(const void* p) { return p && aligned16(p); }

bool sizes_ok(long long B, long long S, long long V) {
    return B > 0 && S > 0 && V > 0 && V < (1ll << 31) && B * S < (1ll << 40);
}

// The launch plan of vocab_rows_kernel: rows [a.row0, a.row0 + a.rows) of a call over N rows cut into chunks of
// chunk_rows (a whole tensor is the one chunk row0 = 0, rows = chunk_rows = N).  Every chunk of a call launches the same
// grid (the plan's chunk_rows, not this chunk's rows, caps it), so chunk c's CTAs own partial rows [c * grid,
// (c + 1) * grid); CTAs past the last chunk's rows store zeros.  The chunk that ends the call adds all n_chunks * grid
// rows of partials: GRPO / RLOO's loss term over a.nb = B sequences, everything else over N rows.
template <class Head, class T>
int launch_rows(T, VocabArgs& a, long long chunk_rows, long long N, float* out, size_t ws_bytes, cudaStream_t st) {
    constexpr auto kern = vocab_rows_kernel<T, Head>;
    constexpr int NP = Head::NP;
    const long long nvec_max = (a.V * (long long)sizeof(T) + 15) / 16;
    a.capv = (NP > 0 && a.grad) ? (int)min(nvec_max, (long long)(VOCAB_SMEM_CAP / 16)) : 0;
    const size_t smem = (size_t)a.capv * 16;
    int sms = 0, per_sm = 0;
    if (int rc = resident_ctas<kern>(VOCAB_NT, smem, sms, per_sm)) return rc;
    const long long grid = min((long long)sms * per_sm, chunk_rows);
    if (NP == 0) return launch_k(kern, (int)grid, VOCAB_NT, smem, st, a);
    const long long n_chunks = (N + chunk_rows - 1) / chunk_rows, chunk = a.row0 / chunk_rows;
    if (!ws_partials_fit(n_chunks * grid * NP, ws_bytes)) return B200RL_ERR_WORKSPACE;
    float* ws = a.ws;
    a.ws = ws + chunk * grid * NP;
    if (int rc = launch_k(kern, (int)grid, VOCAB_NT, smem, st, a)) return rc;
    if (a.row0 + a.rows < N) return B200RL_OK;
    FinalizeArgs fa{};
    for (int k = 0; k < NP; ++k) fa.scale[k] = 1.0 / (double)N;
    if (Head::LOSS_OVER_B) fa.scale[0] = 1.0 / (double)a.nb;
    fa.k = NP;
    fa.n_blocks = (int)(n_chunks * grid);
    return launch_finalize(ws, out, fa, st);
}

// The instantiation table of this file's kernels: f(T(), std::bool_constant<ENT>(), std::bool_constant<KL>()) for the
// runtime dtype (fp32 or bf16) and entropy / kl flags; a kernel that takes neither flag ignores them
template <class F>
int with_vocab(int dtype, bool ent, bool kl, F&& f) {
    const auto flags = [&](auto t) {
        if (ent) return kl ? f(t, std::true_type(), std::true_type()) : f(t, std::true_type(), std::false_type());
        return kl ? f(t, std::false_type(), std::true_type()) : f(t, std::false_type(), std::false_type());
    };
    if (dtype == B200RL_DTYPE_F32) return flags(float());
    if (dtype == B200RL_DTYPE_BF16) return flags(__nv_bfloat16());
    return B200RL_ERR_ARG;
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
    a.inv_b = (float)(1.0 / (double)B); a.nb = B;
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<GrpoRow<true, false>>(t, a, a.rows, a.rows, out3, workspace_bytes, (cudaStream_t)stream);
    });
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
    a.inv_b = (float)(1.0 / (double)B); a.nb = B;
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<GrpoRow<false, false>>(t, a, a.rows, a.rows, out3, workspace_bytes, (cudaStream_t)stream);
    });
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
    return with_vocab(dtype, entropy != 0, kl, [&](auto t, auto ent, auto k) {
        return launch_rows<PpoRow<ent, k, false>>(t, a, rows, rows, out5, workspace_bytes, (cudaStream_t)stream);
    });
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
    return with_vocab(dtype, entropy_row != nullptr, false, [&](auto t, auto ent, auto) {
        return launch_rows<PgBwdRow<ent, false>>(t, a, rows, rows, nullptr, 0, (cudaStream_t)stream);
    });
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
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<A2cRow<false>>(t, a, rows, rows, out3, workspace_bytes, (cudaStream_t)stream);
    });
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
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<PgBwdRow<true, true>>(t, a, rows, rows, nullptr, 0, (cudaStream_t)stream);
    });
}

extern "C" int b200rl_token_logp_fwd(int dtype, const void* logits, const long long* index, long long rows, long long V,
                                     float* logp, float* lse, void* stream) {
    if (!sizes_ok(rows, 1, V) || !aligned_logits(logits) || !index || !logp || !lse) return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logits; a.action = index; a.lp = logp; a.lse = lse;
    a.rows = rows; a.S = 1; a.V = V;
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<LogpRow>(t, a, rows, rows, nullptr, 0, (cudaStream_t)stream);
    });
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
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<CoefBwdRow>(t, a, rows, rows, nullptr, 0, (cudaStream_t)stream);
    });
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

// GRPO / RLOO / per-token log p from the lm_head's hidden states, one chunk of token rows per call
// (ding/rl_utils/grpo.py:43-60 and rloo.py:41-62 with log_prob_fn = efficient_method, log_prob_utils.py:29-48, on
// logits = hidden @ lm_weight^T that the caller computes chunk by chunk; the logit_old / logit_ref streams of
// b200rl_grpo_fwd_grad become the per-token logp_old / logp_ref)
extern "C" int b200rl_lm_linear_fwd(int mode, int dtype, void* logits, long long row0, long long rows,
                                    long long chunk_rows, long long V, long long B, long long S, const long long* action,
                                    const float* logp_old, const float* logp_ref, const float* adv, const float* reward,
                                    long long K, const float* weight, float* seq, double clip_ratio, double beta,
                                    float* logp, float* lse, float* out3, int want_grad, float* workspace,
                                    size_t workspace_bytes, void* stream) {
    const long long N = B * S;
    if (!sizes_ok(B, S, V) || rows < 1 || chunk_rows < rows || row0 < 0 || row0 % chunk_rows || row0 + rows > N ||
        !aligned_logits(logits) || !action || !lse)
        return B200RL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    VocabArgs a{};
    a.x[0] = logits; a.action = action + row0; a.lse = lse + row0;
    a.rows = rows; a.S = S; a.V = V;
    if (mode == B200RL_LM_LOGP) {
        if (!logp) return B200RL_ERR_ARG;
        a.lp = logp + row0;
        return with_vocab(dtype, false, false,
                          [&](auto t, auto, auto) { return launch_rows<LogpRow>(t, a, rows, rows, nullptr, 0, st); });
    }
    const bool grpo = mode == B200RL_LM_GRPO;
    if ((!grpo && mode != B200RL_LM_RLOO) || !logp_old || !seq || !out3 || !workspace ||
        (grpo ? (!logp_ref || !adv) : (!reward || K < 1 || K > (1 << 20) || B % K)) ||
        (dtype != B200RL_DTYPE_F32 && dtype != B200RL_DTYPE_BF16))
        return B200RL_ERR_ARG;
    a.adv = adv; a.reward = reward; a.K = (int)K; a.Bp = grpo ? 0 : B / K;
    a.weight = weight; a.seq = seq; a.nb = B; a.row0 = row0; a.ws = workspace;
    if (row0 == 0) {  // the sequence normalisers, ahead of the first chunk
        int sms = 0, per_sm = 0;
        if (int rc = resident_ctas<lm_seq_kernel>(VOCAB_HEAD_NT, 0, sms, per_sm)) return rc;
        if (int rc = launch_k(lm_seq_kernel, (int)min((long long)sms * per_sm, B), VOCAB_HEAD_NT, 0, st, a)) return rc;
    }
    a.weight = weight ? weight + row0 : nullptr;
    a.lp_old = logp_old + row0; a.lp_ref = grpo ? logp_ref + row0 : nullptr; a.lp = logp ? logp + row0 : nullptr;
    a.grad = want_grad ? logits : nullptr;
    a.lo = (float)(1.0 - clip_ratio); a.hi = (float)(1.0 + clip_ratio); a.beta = grpo ? (float)beta : 0.f;
    a.inv_b = (float)(1.0 / (double)B);
    return with_vocab(dtype, false, grpo, [&](auto t, auto, auto k) {
        return launch_rows<GrpoRow<k, true>>(t, a, chunk_rows, N, out3, workspace_bytes, st);
    });
}

// PPO / A2C from the lm_head's hidden states, one chunk of token rows per call (ding/rl_utils/ppo.py:143-230 with
// calculate_kl_div :30-54, and a2c.py:10-44, on logits = hidden @ lm_weight^T that the caller computes chunk by chunk; the
// logit_old / logit_pretrained streams of b200rl_ppo_lm_fwd_grad become the per-token logp_old / logp_pre)
extern "C" int b200rl_lm_linear_pg_fwd(int mode, int dtype, void* logits, long long row0, long long rows,
                                       long long chunk_rows, long long V, long long N, const long long* action,
                                       const float* logp_old, const float* logp_pre, const float* adv,
                                       const float* value, const float* return_, const float* weight, double clip_ratio,
                                       double dual_clip, int kl_type, int entropy, double w_ent, double w_kl,
                                       double w_val, float* dvalue, float* out, int want_grad, float* workspace,
                                       size_t workspace_bytes, void* stream) {
    const bool ppo = mode == B200RL_LM_PPO, kl = logp_pre != nullptr;
    if (!sizes_ok(N, 1, V) || rows < 1 || chunk_rows < rows || row0 < 0 || row0 % chunk_rows || row0 + rows > N ||
        !aligned_logits(logits) || !action || !adv || !out || !workspace ||
        (dtype != B200RL_DTYPE_F32 && dtype != B200RL_DTYPE_BF16) || (!ppo && mode != B200RL_LM_A2C))
        return B200RL_ERR_ARG;
    if (ppo ? (!logp_old || (kl && (kl_type < 1 || kl_type > 3)) || (!kl && w_kl != 0.0) || (!entropy && w_ent != 0.0) ||
               dvalue || w_val != 0.0)
            : (!value || !return_ || logp_old || kl || w_kl != 0.0))
        return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logits; a.grad = want_grad ? logits : nullptr;
    a.action = action + row0; a.adv = adv + row0; a.weight = weight ? weight + row0 : nullptr;
    a.lp_old = ppo ? logp_old + row0 : nullptr; a.lp_ref = kl ? logp_pre + row0 : nullptr;
    a.value = ppo ? nullptr : value + row0; a.ret = ppo ? nullptr : return_ + row0;
    a.grad_value = dvalue ? dvalue + row0 : nullptr;
    a.ws = workspace; a.row0 = row0;
    a.rows = rows; a.S = 1; a.V = V;
    a.lo = (float)(1.0 - clip_ratio); a.hi = (float)(1.0 + clip_ratio); a.dual_clip = (float)dual_clip;
    a.kl_type = kl_type; a.inv_m = (float)(1.0 / (double)N);
    a.w_ent = (float)w_ent; a.w_kl = (float)w_kl; a.w_val = (float)w_val;
    cudaStream_t st = (cudaStream_t)stream;
    if (!ppo)
        return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
            return launch_rows<A2cRow<true>>(t, a, chunk_rows, N, out, workspace_bytes, st);
        });
    return with_vocab(dtype, entropy != 0, kl, [&](auto t, auto ent, auto k) {
        return launch_rows<PpoRow<ent, k, true>>(t, a, chunk_rows, N, out, workspace_bytes, st);
    });
}

// The backward of token_logp_linear on one chunk, in place (log_prob_utils.py:29-48's autograd, as b200rl_token_logp_bwd)
extern "C" int b200rl_lm_linear_bwd(int dtype, void* logits, long long row0, long long rows, long long V,
                                    const long long* index, const float* lse, const float* dlogp, void* stream) {
    if (!sizes_ok(rows, 1, V) || row0 < 0 || !aligned_logits(logits) || !index || !lse || !dlogp) return B200RL_ERR_ARG;
    VocabArgs a{};
    a.x[0] = logits; a.grad = logits;
    a.action = index + row0; a.lse = const_cast<float*>(lse + row0); a.coef_in = dlogp + row0;
    a.rows = rows; a.S = 1; a.V = V;
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        return launch_rows<CoefBwdRow>(t, a, rows, rows, nullptr, 0, (cudaStream_t)stream);
    });
}

extern "C" int b200rl_lm_linear_scale(int dtype, const float* g, void* x, long long n, void* stream) {
    if (n < 0 || !g || (n > 0 && (!x || !aligned16(x)))) return B200RL_ERR_ARG;
    if (n == 0) return B200RL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        using T = decltype(t);
        int sms = 0, per_sm = 0;
        if (int rc = resident_ctas<scale_inplace_kernel<T>>(256, 0, sms, per_sm)) return rc;
        const long long grid = min((long long)sms * per_sm, (n / VecT<T>::W + 255) / 256 + 1);
        return launch_k(scale_inplace_kernel<T>, (int)grid, 256, 0, st, g, (T*)x, n);
    });
}

extern "C" int b200rl_lm_linear_scale_out(int dtype, const float* g, const void* in, void* out, long long n,
                                          void* stream) {
    if (n < 0 || !g || (n > 0 && (!in || !out || !aligned16(in) || !aligned16(out)))) return B200RL_ERR_ARG;
    if (n == 0) return B200RL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    return with_vocab(dtype, false, false, [&](auto t, auto, auto) {
        using T = decltype(t);
        int sms = 0, per_sm = 0;
        if (int rc = resident_ctas<scale_out_kernel<T>>(256, 0, sms, per_sm)) return rc;
        const long long grid = min((long long)sms * per_sm, (n / VecT<T>::W + 255) / 256 + 1);
        return launch_k(scale_out_kernel<T>, (int)grid, 256, 0, st, g, (const T*)in, (T*)out, n);
    });
}
