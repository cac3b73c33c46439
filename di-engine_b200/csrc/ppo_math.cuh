#pragma once
// Shared device code of the PPO tile kernels (ppo.cu) and the fused one-pass learner step (fused.cu).
#include "common.cuh"

namespace b200rl {

struct PpoArgs {
    const float* logit_new;
    const float* logit_old;
    const float* logit_pre;  // nullable
    const long long* action;
    const float* value_new;
    const float* value_old;
    const float* adv;
    float* adv_out;  // fused learner step only: where phase G writes the advantage (same buffer as adv)
    const float* ret;
    const float* weight;  // nullable -> 1
    long long S;
    int G;
    int N;
    float clip;       // fp32(clip_ratio)
    float clip_lo;    // fp32(1 - clip_ratio), computed in double like the python scalar of the reference
    float clip_hi;    // fp32(1 + clip_ratio)
    float dual_clip;  // <= 0: disabled
    int use_value_clip;
    int kl_type;  // 1,2,3
    float* grad_logit;
    float* grad_value;
    UpstreamRecord rec;  // FWD_GRAD and BWD (ppo_owned slots)
    // nullable: {mean, std + 1e-8} of the advantage batch (device floats, b200rl_adv_stats): when given every kernel uses
    // (adv - mean) / (std + 1e-8) -- PPOPolicy's per-batch advantage normalisation (ding/policy/ppo.py:304-306) applied on load
    const float* adv_stats;
    // nullable, (S): happo_error's per-sample factor (the other agents' ratio product, ding/rl_utils/happo.py:124-125): the
    // selected surrogate is multiplied by it before the dual clip
    const float* factor;
};

// d(selected surrogate)/d(ratio) with torch's tie rules: min/max split the gradient 0.5/0.5 on equality, clamp passes
// gradient on the closed interval (ppo.py:208-216).  Also returns the selected surrogate value.
// dual_all: ppo_error_continuous applies max(., dual_clip * adv) to EVERY sample (ppo.py:346-347), the discrete loss only where
// adv < 0 (ppo.py:211-214)
// fac: happo's factor multiplies min(surr1, surr2) before the dual clip (happo.py:124-130); 1 for every PPO loss
__device__ __forceinline__ float surrogate(float ratio, float adv, float lo, float hi, float dual_clip,
                                           float& dsel_dratio, bool dual_all = false, float fac = 1.f) {
    const float rc = fminf(fmaxf(ratio, lo), hi);
    const float s1 = ratio * adv, s2 = rc * adv;
    const float in_range = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
    float w1, w2;
    if (s1 < s2) { w1 = 1.f; w2 = 0.f; }
    else if (s1 > s2) { w1 = 0.f; w2 = 1.f; }
    else { w1 = 0.5f; w2 = 0.5f; }
    float sel = fminf(s1, s2) * fac;
    float d = adv * (w1 + w2 * in_range) * fac;
    if (dual_clip > 0.f && (dual_all || adv < 0.f)) {
        const float floor_ = dual_clip * adv;
        if (sel < floor_) { sel = floor_; d = 0.f; }
        else if (sel == floor_) { d *= 0.5f; }
    }
    dsel_dratio = d;
    return sel;
}

// 0.5*w*max(e1,e2) pieces: returns max(e1,e2) and d max / d value_new (ppo.py:267-274)
__device__ __forceinline__ float value_term(float v, float v_old, float ret, float clip, int use_clip, float& dterm_dv) {
    const float r1 = ret - v;
    const float e1 = r1 * r1;
    if (!use_clip) { dterm_dv = -2.f * r1; return e1; }
    const float dv = v - v_old;
    const float vc = v_old + fminf(fmaxf(dv, -clip), clip);
    const float r2 = ret - vc;
    const float e2 = r2 * r2;
    const float pass = (dv >= -clip && dv <= clip) ? 1.f : 0.f;
    const float d1 = -2.f * r1, d2 = -2.f * r2 * pass;
    if (e1 > e2) { dterm_dv = d1; return e1; }
    if (e1 < e2) { dterm_dv = d2; return e2; }
    dterm_dv = 0.5f * (d1 + d2);
    return e1;
}

// ===============================================================================================================
// main path: persistent TMA-pipelined tile kernel
// ===============================================================================================================
constexpr int PPO_CW = 4;                       // consumer warps per CTA
constexpr int PPO_CT = PPO_CW * 32;            // consumer threads per CTA
constexpr int PPO_THREADS = PPO_CT + 32;      // + one producer warp
constexpr int PPO_STAGES = 3;   // input ring depth
constexpr int PPO_OUTBUFS = 2;  // gradient tile ring depth (per warp)
enum { PPO_FWD = 0, PPO_FWD_GRAD = 1, PPO_BWD = 2 };

// MUFU approximations with flush-to-zero (no denormal fix-up code around them): relative error ~2^-22
__device__ __forceinline__ float ex2f_(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2f_(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcpf_(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kF32Min = -3.402823466e38f;
// Floor of t_j = (z_j - max)*log2(e) in the tile kernels.  2^t_j is already 0 in fp32 far above it, so it changes no
// probability and no entropy term (Categorical.entropy clamps log p at finfo.min for the same reason: a -inf logit must
// give 0, not 0 * -inf).  Unlike finfo.min it keeps k1*t_j finite in the gradient factor p_j*(k0 - k1*t_j) for any
// |k1| < 1e36, so a masked logit (p_j = 0) gets an exact 0 even when |k1| = |g_ent*w*ln2/S| > 1.
constexpr float kT2Min = -256.f;

// advantage as the loss sees it: raw, or normalised with the batch statistics (two fp32 ops, as torch evaluates the expression)
__device__ __forceinline__ float adv_in(const PpoArgs& a, float adv) {
    return a.adv_stats ? __fdiv_rn(fsub(adv, a.adv_stats[0]), a.adv_stats[1]) : adv;
}

__device__ __forceinline__ float kl_term(float log_ratio, int kl_type, float& dterm) {
    if (kl_type == 1) { dterm = 1.f; return log_ratio; }
    if (kl_type == 2) { dterm = log_ratio; return log_ratio * log_ratio / 2.f; }
    const float e = ex2f_(-log_ratio * kLog2e);
    dterm = 1.f - e;
    return e - 1.f + log_ratio;
}

// one row of NC logits from shared memory into registers; 8/16-byte vector loads are bank-conflict free for the
// row strides that occur (e.g. 24 B rows read as 3 x float2)
template <int NC>
__device__ __forceinline__ void load_row(const float* src, float (&z)[NC]) {
    if (NC % 4 == 0) {
#pragma unroll
        for (int j = 0; j < NC / 4; ++j) {
            const float4 v = reinterpret_cast<const float4*>(src)[j];
            z[4 * j] = v.x; z[4 * j + 1] = v.y; z[4 * j + 2] = v.z; z[4 * j + 3] = v.w;
        }
    } else if (NC % 2 == 0) {
#pragma unroll
        for (int j = 0; j < NC / 2; ++j) {
            const float2 v = reinterpret_cast<const float2*>(src)[j];
            z[2 * j] = v.x; z[2 * j + 1] = v.y;
        }
    } else {
#pragma unroll
        for (int j = 0; j < NC; ++j) z[j] = src[j];
    }
}
template <int NC>
__device__ __forceinline__ void store_row(float* dst, const float (&g)[NC]) {
    if (NC % 4 == 0) {
#pragma unroll
        for (int j = 0; j < NC / 4; ++j)
            reinterpret_cast<float4*>(dst)[j] = make_float4(g[4 * j], g[4 * j + 1], g[4 * j + 2], g[4 * j + 3]);
    } else if (NC % 2 == 0) {
#pragma unroll
        for (int j = 0; j < NC / 2; ++j) reinterpret_cast<float2*>(dst)[j] = make_float2(g[2 * j], g[2 * j + 1]);
    } else {
#pragma unroll
        for (int j = 0; j < NC; ++j) dst[j] = g[j];
    }
}

// Softmax statistics of one row in the log2 domain: t_j = (z_j - max)*log2(e) <= 0, e_j = 2^t_j, s = sum e_j,
// u2 = sum e_j t_j.  Then logsumexp = max + ln2*log2(s), entropy = ln2*(log2(s) - u2/s), p_j = e_j/s.
struct RowStat {
    float m, l2s, inv, log_s, ent;
};

struct PpoTileLayout {
    int logit_bytes;  // one logit tile
    int off_old, off_pre, off_act, off_vn, off_vo, off_adv, off_ret, off_w;
    int stage_bytes;
    int tx_bytes;  // bytes TMA delivers per stage
};
__host__ __device__ inline PpoTileLayout ppo_layout(int N, bool has_pre, bool has_w, int PPO_R) {
    PpoTileLayout L;
    L.logit_bytes = PPO_R * N * 4;
    int o = L.logit_bytes;
    L.off_old = o; o += L.logit_bytes;
    L.off_pre = o; if (has_pre) o += L.logit_bytes;
    L.off_act = o; o += PPO_R * 8;
    L.off_vn = o; o += PPO_R * 4;
    L.off_vo = o; o += PPO_R * 4;
    L.off_adv = o; o += PPO_R * 4;
    L.off_ret = o; o += PPO_R * 4;
    L.off_w = o; if (has_w) o += PPO_R * 4;
    L.stage_bytes = (o + 127) & ~127;
    L.tx_bytes = o;
    return L;
}


struct PpoUpstream {
    float g_pol, g_val, g_ent, g_kl, inv_s;
};

// slots of the upstream-gradient record a PPO kernel owns: policy, value, entropy, and kl with logit_pretrained
__device__ __forceinline__ unsigned ppo_owned(const PpoArgs& a) { return a.logit_pre ? 15u : 7u; }

// One row (thread = row `tid` of the tile staged at `st`): softmax statistics, clipped surrogate, value term, optional
// KL, loss partial sums (LOSSES) and the gradient row (GRADS; into the shared-memory tile `gtile` for full tiles, straight
// to global memory for the ragged last tile).  `adv` is passed by value (staged by TMA in ppo.cu, read from L2 right
// after the GAE scan produced it in fused.cu).  The destinations are explicit: `gr` receives the row's N logit gradients
// (it may alias the row's own logit_new slot in `st`: every read of that slot precedes the write) and `gv` the value
// gradient.
template <int NC, bool LOSSES, bool GRADS>
__device__ __forceinline__ void ppo_row_compute_to(const PpoArgs& a, const PpoTileLayout& L, const unsigned char* st,
                                                   int tid, int N, float adv, float* gr, float* gv,
                                                   const PpoUpstream& up, float (&acc)[6], float fac = 1.f) {
    adv = adv_in(a, adv);
    const bool has_pre = a.logit_pre != nullptr, has_w = a.weight != nullptr;
    const float g_pol = up.g_pol, g_val = up.g_val, g_ent = up.g_ent, g_kl = up.g_kl, inv_s = up.inv_s;
    {
            const float* zn = reinterpret_cast<const float*>(st) + tid * N;
            const float* zo = reinterpret_cast<const float*>(st + L.off_old) + tid * N;
            const int act = (int)reinterpret_cast<const long long*>(st + L.off_act)[tid];
            const float v_new = reinterpret_cast<const float*>(st + L.off_vn)[tid];
            const float v_old = reinterpret_cast<const float*>(st + L.off_vo)[tid];
            const float ret = reinterpret_cast<const float*>(st + L.off_ret)[tid];
            const float w = has_w ? reinterpret_cast<const float*>(st + L.off_w)[tid] : 1.f;
            constexpr int NR = NC ? NC : 1;
            float tn[NR], en[NR];  // new-policy row: t_j and e_j (compile-time N only)
            float m = kF32Min, s = 0.f, u2 = 0.f;
            if (NC) {
                load_row<NR>(zn, tn);
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
                for (int j = 0; j < N; ++j) m = fmaxf(m, zn[j]);
                const float m2 = m * kLog2e;
                for (int j = 0; j < N; ++j) {
                    const float t = fmaxf(fmaf(zn[j], kLog2e, -m2), kT2Min);
                    const float e = ex2f_(t);
                    s += e;
                    u2 = fmaf(e, t, u2);
                }
            }
            const float l2s = lg2f_(s), inv_sum = rcpf_(s);
            const float log_s = l2s * kLn2;
            const float ent = (l2s - u2 * inv_sum) * kLn2;
            const float lp_n = (zn[act] - m) - log_s;
            // behaviour ("old") policy row: only logsumexp is needed
            float mo = kF32Min, so = 0.f;
            if (NC) {
                float to[NR];
                load_row<NR>(zo, to);
#pragma unroll
                for (int j = 0; j < NR; ++j) mo = fmaxf(mo, to[j]);
                const float mo2 = mo * kLog2e;
#pragma unroll
                for (int j = 0; j < NR; ++j) so += ex2f_(fmaf(to[j], kLog2e, -mo2));
            } else {
                for (int j = 0; j < N; ++j) mo = fmaxf(mo, zo[j]);
                const float mo2 = mo * kLog2e;
                for (int j = 0; j < N; ++j) so += ex2f_(fmaf(zo[j], kLog2e, -mo2));
            }
            const float lp_o = (zo[act] - mo) - lg2f_(so) * kLn2;
            const float ratio = ex2f_((lp_n - lp_o) * kLog2e);
            float dsel, dterm, dk = 0.f, klv = 0.f;
            const float sel = surrogate(ratio, adv, a.clip_lo, a.clip_hi, a.dual_clip, dsel, false, fac);
            const float vt = value_term(v_new, v_old, ret, a.clip, a.use_value_clip, dterm);
            if (has_pre) {
                const float* zp = reinterpret_cast<const float*>(st + L.off_pre) + tid * N;
                float mp = kF32Min, sp = 0.f;
                for (int j = 0; j < N; ++j) mp = fmaxf(mp, zp[j]);
                const float mp2 = mp * kLog2e;
                for (int j = 0; j < N; ++j) sp += ex2f_(fmaf(zp[j], kLog2e, -mp2));
                klv = kl_term(lp_n - ((zp[act] - mp) - lg2f_(sp) * kLn2), a.kl_type, dk);
            }
            if (LOSSES) {
                acc[0] -= sel * w;
                acc[1] += vt * w;
                acc[2] += ent * w;
                acc[3] += klv;
                acc[4] += lp_o - lp_n;
                acc[5] += (ratio > a.clip_hi || ratio < a.clip_lo) ? 1.f : 0.f;
            }
            if (GRADS) {
                // d/dlogp(a): policy -(w/S)*dsel*ratio, kl dk/S;  d/dH: entropy w/S
                const float c_act = g_pol * (-w * inv_s) * dsel * ratio + g_kl * dk * inv_s;
                const float c_ent = g_ent * w * inv_s;
                // grad z_j = c_act*(1[j==a] - p_j) - c_ent*p_j*(logp_j + H),  logp_j = ln2*t_j - log_s
                //          = p_j*(k0 - k1*t_j) + 1[j==a]*c_act
                const float k0 = -c_act - c_ent * (ent - log_s), k1 = c_ent * kLn2;
                if (NC) {
                    float gj[NR];
#pragma unroll
                    for (int j = 0; j < NR; ++j) {
                        gj[j] = (en[j] * inv_sum) * fmaf(-k1, tn[j], k0);
                        if (j == act) gj[j] += c_act;
                    }
                    store_row<NR>(gr, gj);  // 8/16-byte vector stores: rows are N*4 bytes apart from a 16-byte aligned base
                } else {
                    const float m2 = m * kLog2e;
                    for (int j = 0; j < N; ++j) {
                        const float t = fmaxf(fmaf(zn[j], kLog2e, -m2), kT2Min);
                        float g = (ex2f_(t) * inv_sum) * fmaf(-k1, t, k0);
                        if (j == act) g += c_act;
                        gr[j] = g;
                    }
                }
                *gv = g_val * 0.5f * w * inv_s * dterm;
            }
        }
}

// row `tid` of a tile of consecutive rows starting at global row `row0` (ppo.cu, fused.cu)
template <int NC, bool LOSSES, bool GRADS>
__device__ __forceinline__ void ppo_row_compute(const PpoArgs& a, const PpoTileLayout& L, const unsigned char* st,
                                                int tid, int N, float adv, bool full_tile, float* gtile,
                                                long long row0, const PpoUpstream& up, float (&acc)[6]) {
    float* gr = GRADS ? (full_tile ? gtile + tid * N : a.grad_logit + (row0 + tid) * N) : nullptr;
    float* gv = GRADS ? a.grad_value + row0 + tid : nullptr;
    ppo_row_compute_to<NC, LOSSES, GRADS>(a, L, st, tid, N, adv, gr, gv, up, acc, a.factor ? a.factor[row0 + tid] : 1.f);
}

}  // namespace b200rl
