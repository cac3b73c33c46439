// PPO clipped surrogate + value + entropy (+ optional KL-to-pretrained) loss, forward and backward.
// Replaces ppo_error / ppo_policy_error / ppo_value_error of ding/rl_utils/ppo.py:77-275 (~40 torch kernels forward
// plus the autograd backward, and two .item() host syncs).
//
// Shapes: S samples, G "agent" rows per sample (G == 1 except the multi-agent case ppo.py:199-200,206-207),
// N logits per row.  logit_* are (S*G, N) row-major, action (S*G) int64, value_new/value_old/adv/return_/weight (S).
//
// Main path (G == 1, N <= 32, 16-byte aligned tensors): ppo_tile_kernel
//   * persistent grid (SM count x resident CTAs), each CTA walks tiles of 128 consecutive rows;
//   * every input of a tile -- the logit rows (128*N contiguous floats per tensor), the int64 actions and the four
//     per-sample scalars -- arrives in shared memory by TMA 1-D bulk copies (cp.async.bulk, SASS UBLKCP) that complete
//     on an mbarrier; a 3-stage ring keeps two tiles in flight per CTA while one is consumed, so HBM latency is hidden
//     without spending issue slots on address arithmetic;
//   * thread i owns row i of the tile; N is a template parameter (rows live in registers, loops fully unrolled) and the
//     softmax statistics use ex2/lg2 approximations (relative error ~1e-7, far inside the 1e-5 parity bar);
//   * gradient tiles leave through shared memory and TMA bulk stores (cp.async.bulk.global.shared::cta);
//   * loss partial sums stay in registers across tiles; one deterministic grid reduction per CTA at the end.
//   Three variants of the same pipeline: FWD (losses), BWD (gradients for given upstream gradients) and FWD_GRAD: the
//   forward pass also writes the gradients for the upstream gradients it is told to expect (they are constants of the
//   training loop: policy + c_v*value - c_e*entropy), so the batch crosses HBM once; the backward launch then only
//   verifies the expectation on the device and recomputes nothing unless it was wrong (exact for any upstream value).
// Fallback paths: DIRECT L=1 one thread per sample (multi-agent / unaligned / N in 33..64), DIRECT L=32 one warp per
// sample (large N, e.g. token vocabularies).
//
// Forward output: out[0..5] = policy_loss, value_loss, entropy_loss, kl_div, approx_kl, clipfrac (device floats, the
// caller decides when to read them -- no host sync in here).
#include "../../include/b200rl.h"
#include "ppo_math.cuh"

namespace b200rl {

template <int NC, int WHAT>
__global__ void __launch_bounds__(PPO_THREADS) ppo_tile_kernel(PpoArgs a, float* out, float* ws) {
    // rows per tile: one per consumer thread (256-row tiles can help the forward-only variant, not the gradient-writing
    // ones or the gae -> ppo -> verify sequence)
    constexpr int PPO_R = PPO_CT;
    pdl_prologue();
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr bool GRADS = (WHAT != PPO_FWD);
    constexpr bool LOSSES = (WHAT != PPO_BWD);
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x;
    const int wid = tid >> 5, lane = tid & 31;
    const bool is_producer = wid == PPO_CW;  // warp 4: TMA issue only
    const bool has_pre = a.logit_pre != nullptr, has_w = a.weight != nullptr;
    const PpoTileLayout L = ppo_layout(N, has_pre, has_w, PPO_R);
    const int warp_out_bytes = 32 * N * 4;  // one warp's gradient rows of a tile (32 consecutive rows)
    unsigned char* outbuf = smem + PPO_STAGES * L.stage_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + (GRADS ? PPO_OUTBUFS * L.logit_bytes : 0));
    uint64_t* empty = full + PPO_STAGES;

    float g[4] = {0.f, 0.f, 0.f, 0.f};
    // BWD: returns when the forward pass wrote exactly these gradients
    if (GRADS && upstream<4>(a.rec, WHAT == PPO_BWD, ppo_owned(a), g)) return;
    const PpoUpstream up{g[0], g[1], g[2], g[3], 1.f / (float)a.S};

    const long long n_full = a.S / PPO_R;
    const int tail_rows = (int)(a.S - n_full * PPO_R);
    const long long n_tiles = n_full + (tail_rows ? 1 : 0);
    const int my_n = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;

    if (tid == 0) {
        for (int s = 0; s < PPO_STAGES; ++s) {
            mbar_init(&full[s], 1);           // producer's expect_tx arrive + TMA byte count
            mbar_init(&empty[s], PPO_CW);  // one arrive per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // policy, value, entropy, kl, approx_kl, clipfrac
    if (is_producer) {
        // ---- producer warp: keeps the stage ring full; never touches the data ---------------------------------------
        if (lane == 0) {
            for (int i = 0; i < my_n; ++i) {
                const long long t = blockIdx.x + (long long)i * gridDim.x;
                if (t >= n_full) break;  // the ragged last tile is read with plain loads by its consumers
                const int sg = i % PPO_STAGES;
                if (i >= PPO_STAGES) mbar_wait(&empty[sg], (uint32_t)(((i / PPO_STAGES) - 1) & 1));
                const long long row0 = t * PPO_R;
                unsigned char* st = smem + sg * L.stage_bytes;
                uint64_t* bar = &full[sg];
                mbar_expect_tx(bar, (uint32_t)L.tx_bytes);
                tma_load_1d(st, a.logit_new + row0 * N, L.logit_bytes, bar);
                tma_load_1d(st + L.off_old, a.logit_old + row0 * N, L.logit_bytes, bar);
                if (has_pre) tma_load_1d(st + L.off_pre, a.logit_pre + row0 * N, L.logit_bytes, bar);
                tma_load_1d(st + L.off_act, a.action + row0, PPO_R * 8, bar);
                tma_load_1d(st + L.off_vn, a.value_new + row0, PPO_R * 4, bar);
                tma_load_1d(st + L.off_vo, a.value_old + row0, PPO_R * 4, bar);
                tma_load_1d(st + L.off_adv, a.adv + row0, PPO_R * 4, bar);
                tma_load_1d(st + L.off_ret, a.ret + row0, PPO_R * 4, bar);
                if (has_w) tma_load_1d(st + L.off_w, a.weight + row0, PPO_R * 4, bar);
            }
        }
    } else {
    // ---- consumer warps: warp w owns rows [32w, 32w+32) of every tile; no CTA-wide barrier in this loop ------------
    const int rit = wid * 32 + lane;  // this thread's row in every tile
    for (int i = 0; i < my_n; ++i) {
        const long long t = blockIdx.x + (long long)i * gridDim.x;
        const long long row0 = t * PPO_R;
        const int sg = i % PPO_STAGES;
        unsigned char* st = smem + sg * L.stage_bytes;
        const bool full_tile = t < n_full;
        if (full_tile) {
            mbar_wait(&full[sg], (uint32_t)((i / PPO_STAGES) & 1));
        } else {
            // ragged last tile: every thread fetches its own row into its own slots of the stage (no sharing)
            if (rit < tail_rows) {
                float* d0 = reinterpret_cast<float*>(st) + rit * N;
                float* d1 = reinterpret_cast<float*>(st + L.off_old) + rit * N;
                float* d2 = reinterpret_cast<float*>(st + L.off_pre) + rit * N;
                for (int k = 0; k < N; ++k) {
                    d0[k] = a.logit_new[(row0 + rit) * N + k];
                    d1[k] = a.logit_old[(row0 + rit) * N + k];
                    if (has_pre) d2[k] = a.logit_pre[(row0 + rit) * N + k];
                }
                reinterpret_cast<long long*>(st + L.off_act)[rit] = a.action[row0 + rit];
                reinterpret_cast<float*>(st + L.off_vn)[rit] = a.value_new[row0 + rit];
                reinterpret_cast<float*>(st + L.off_vo)[rit] = a.value_old[row0 + rit];
                reinterpret_cast<float*>(st + L.off_adv)[rit] = a.adv[row0 + rit];
                reinterpret_cast<float*>(st + L.off_ret)[rit] = a.ret[row0 + rit];
                if (has_w) reinterpret_cast<float*>(st + L.off_w)[rit] = a.weight[row0 + rit];
            }
        }
        // this warp's slice of the gradient-tile ring (2 buffers per warp inside the CTA's output area)
        float* gtile = reinterpret_cast<float*>(outbuf + (wid * 2 + (i & 1)) * warp_out_bytes) - wid * 32 * N;
        if (full_tile || rit < tail_rows) {
            const float adv = reinterpret_cast<const float*>(st + L.off_adv)[rit];
            ppo_row_compute<NC, LOSSES, GRADS>(a, L, st, rit, N, adv, full_tile, gtile, row0, up, acc);
        }
        if (full_tile) {
            if (GRADS) {
                // hand this warp's 32 gradient rows to the TMA store engine; keep at most one store reading smem
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                    tma_store_1d(a.grad_logit + (row0 + wid * 32) * N, gtile + wid * 32 * N, warp_out_bytes);
                    tma_store_commit();
                    tma_store_wait_read<1>();
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[sg]);  // stage may be refilled once all four warps have arrived
        }
    }
    if (GRADS && lane == 0) tma_store_wait_read<0>();  // shared memory must outlive the bulk stores that read it
    }
    if (LOSSES) grid_store_partials<6, PPO_THREADS>(acc, ws);  // summed by finalize_sums_kernel, launched right behind
}

// ===============================================================================================================
// fallback paths (multi-agent rows, N > 32, unaligned tensors): direct global loads
// ===============================================================================================================
// MODE 1: one thread per sample, 2: one warp per sample
template <int NT, int MODE>
__global__ void __launch_bounds__(NT) ppo_fwd_kernel(PpoArgs a, float* out, float* ws) {
    pdl_prologue();
    constexpr int L = (MODE == 2) ? 32 : 1;
    const int lane = (MODE == 2) ? (threadIdx.x & 31) : 0;
    const int N = a.N, G = a.G;
    // grid-stride over the samples: the grid (and with it the per-CTA partial sums in the workspace) is capped by the host
    const long long per_cta = (MODE == 1) ? NT : NT / 32;
    long long s = (MODE == 1) ? (long long)blockIdx.x * NT + threadIdx.x
                              : (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // policy, value, entropy, kl, approx_kl, clipfrac
    for (; s < a.S; s += per_cta * gridDim.x) {
        const float* zn = a.logit_new + s * G * N;
        const float* zo = a.logit_old + s * G * N;
        const float* zp = a.logit_pre ? a.logit_pre + s * G * N : nullptr;
        float ratio_sum = 0.f, ent_sum = 0.f, akl = 0.f, kl = 0.f;
        for (int g = 0; g < G; ++g) {
            const float* rn = zn + (size_t)g * N;
            const float* ro = zo + (size_t)g * N;
            const int act = (int)a.action[s * G + g];
            float lse_n, ent;
            row_lse_entropy<L>([&](int j) { return rn[j]; }, N, lane, lse_n, ent);
            const float lse_o = row_lse<L>([&](int j) { return ro[j]; }, N, lane);
            const float lp_n = rn[act] - lse_n;
            const float lp_o = ro[act] - lse_o;
            ratio_sum += expf(lp_n - lp_o);
            ent_sum += ent;
            akl += lp_o - lp_n;
            if (zp) {
                const float* rp = zp + (size_t)g * N;
                const float lse_p = row_lse<L>([&](int j) { return rp[j]; }, N, lane);
                float dummy;
                kl += kl_term(lp_n - (rp[act] - lse_p), a.kl_type, dummy);
            }
        }
        if (lane == 0) {
            const float w = a.weight ? a.weight[s] : 1.f;
            const float adv = adv_in(a, a.adv[s]);
            const float ratio = (G == 1) ? ratio_sum : ratio_sum / (float)G;
            const float ent = (G == 1) ? ent_sum : ent_sum / (float)G;
            float dsel;
            const float sel = surrogate(ratio, adv, a.clip_lo, a.clip_hi, a.dual_clip, dsel, false, a.factor ? a.factor[s] : 1.f);
            acc[0] -= sel * w;
            float dterm;
            acc[1] += value_term(a.value_new[s], a.value_old[s], a.ret[s], a.clip, a.use_value_clip, dterm) * w;
            acc[2] += ent * w;
            acc[3] += kl;
            acc[4] += akl;
            acc[5] += (ratio > a.clip_hi || ratio < a.clip_lo) ? 1.f : 0.f;
        }
    }
    double tot[6];
    if (grid_sum<6, NT>(acc, tot, ws, 0) && threadIdx.x == 0) {
        const double inv_s = 1.0 / (double)a.S, inv_m = 1.0 / ((double)a.S * (double)G);
        out[0] = (float)(tot[0] * inv_s);
        out[1] = (float)(0.5 * tot[1] * inv_s);
        out[2] = (float)(tot[2] * inv_s);
        out[3] = a.logit_pre ? (float)(tot[3] * inv_m) : 0.f;
        out[4] = (float)(tot[4] * inv_m);
        out[5] = (float)(tot[5] * inv_s);
    }
}

template <int NT, int MODE>
__global__ void __launch_bounds__(NT) ppo_bwd_kernel(PpoArgs a) {
    pdl_prologue();
    constexpr int L = (MODE == 2) ? 32 : 1;
    const int lane = (MODE == 2) ? (threadIdx.x & 31) : 0;
    const int N = a.N, G = a.G;
    // reads the upstream gradients and refreshes the hint; the host never passes a `used` record here (the fused forward
    // exists on the tile path only), so this launch always computes
    float g[4];
    upstream<4>(a.rec, true, ppo_owned(a), g);
    const float g_pol = g[0], g_val = g[1], g_ent = g[2], g_kl = g[3];
    const float inv_s = 1.f / (float)a.S;
    const float inv_m = 1.f / ((float)a.S * (float)G);
    const long long per_cta = (MODE == 1) ? NT : NT / 32;
    long long s = (MODE == 1) ? (long long)blockIdx.x * NT + threadIdx.x
                              : (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
    for (; s < a.S; s += per_cta * gridDim.x) {
    const float* zn = a.logit_new + s * G * N;
    const float* zo = a.logit_old + s * G * N;
    const float* zp = a.logit_pre ? a.logit_pre + s * G * N : nullptr;
    float* gz = a.grad_logit + s * G * N;
    const float w = a.weight ? a.weight[s] : 1.f;
    const float adv = adv_in(a, a.adv[s]);
    // pass A (only when G > 1): the sample's mean ratio decides the clip branch for all of its rows
    float ratio_s = 0.f;
    if (G > 1) {
        for (int g = 0; g < G; ++g) {
            const float* rn = zn + (size_t)g * N;
            const float* ro = zo + (size_t)g * N;
            const int act = (int)a.action[s * G + g];
            const float lse_n = row_lse<L>([&](int j) { return rn[j]; }, N, lane);
            const float lse_o = row_lse<L>([&](int j) { return ro[j]; }, N, lane);
            ratio_s += expf((rn[act] - lse_n) - (ro[act] - lse_o));
        }
        ratio_s /= (float)G;
    }
    for (int g = 0; g < G; ++g) {
        const float* rn = zn + (size_t)g * N;
        const float* ro = zo + (size_t)g * N;
        float* gr = gz + (size_t)g * N;
        const int act = (int)a.action[s * G + g];
        float lse_n, ent;
        row_lse_entropy<L>([&](int j) { return rn[j]; }, N, lane, lse_n, ent);
        const float lse_o = row_lse<L>([&](int j) { return ro[j]; }, N, lane);
        const float lp_n = rn[act] - lse_n;
        const float ratio_g = expf(lp_n - (ro[act] - lse_o));
        if (G == 1) ratio_s = ratio_g;
        float dsel;
        surrogate(ratio_s, adv, a.clip_lo, a.clip_hi, a.dual_clip, dsel, false, a.factor ? a.factor[s] : 1.f);
        // d policy_loss / d logp_new(row) = -(w/S) * dsel/dratio * ratio_g / G
        float c_act = g_pol * (-w * inv_s) * dsel * ratio_g / (float)G;
        if (zp) {
            const float* rp = zp + (size_t)g * N;
            const float lse_p = row_lse<L>([&](int j) { return rp[j]; }, N, lane);
            float dk;
            kl_term(lp_n - (rp[act] - lse_p), a.kl_type, dk);
            c_act += g_kl * dk * inv_m;
        }
        const float c_ent = g_ent * w * inv_m;  // d entropy_loss / d H(row)
        // grad z_j = c_act*(1[j==a] - p_j) - c_ent * p_j*(logp_j + H)
        for (int j = lane; j < N; j += L) {
            const float lp = fmaxf(rn[j] - lse_n, kF32Min);  // Categorical.entropy's clamp: 0 * finite at a -inf logit
            const float p = expf(lp);
            float gj = -c_act * p - c_ent * p * (lp + ent);
            if (j == act) gj += c_act;
            gr[j] = gj;
        }
    }
    if (lane == 0) {
        float dterm;
        value_term(a.value_new[s], a.value_old[s], a.ret[s], a.clip, a.use_value_clip, dterm);
        a.grad_value[s] = g_val * 0.5f * w * inv_s * dterm;
    }
    }
}

static bool tile_path_ok(const PpoArgs& a) {
    const bool al = aligned16(a.logit_new) && aligned16(a.logit_old) && (!a.logit_pre || aligned16(a.logit_pre)) &&
                    aligned16(a.action) && aligned16(a.value_new) && aligned16(a.value_old) && aligned16(a.adv) &&
                    aligned16(a.ret) && (!a.weight || aligned16(a.weight)) &&
                    (!a.grad_logit || aligned16(a.grad_logit));
    return a.G == 1 && a.N <= 32 && al;
}

// ppo_value_error alone (ppo.py:233-275; PPG's auxiliary phase and value-only updates call it without the policy part):
// value loss and its gradient for a unit upstream gradient in one pass; backward is a scale of the saved gradient.
template <int NT>
__global__ void __launch_bounds__(NT) ppo_value_kernel(const float* __restrict__ value_new,
                                                       const float* __restrict__ value_old,
                                                       const float* __restrict__ ret, const float* __restrict__ weight,
                                                       long long S, float clip, int use_clip, float* __restrict__ out,
                                                       float* __restrict__ dvalue, float* ws) {
    pdl_prologue();
    float acc[1] = {0.f};
    const float inv_s = 1.f / (float)S;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < S; i += (long long)gridDim.x * NT) {
        const float w = weight ? weight[i] : 1.f;
        float d;
        const float t = value_term(value_new[i], use_clip ? value_old[i] : 0.f, ret[i], clip, use_clip, d);
        acc[0] += t * w;
        if (dvalue) dvalue[i] = 0.5f * w * inv_s * d;
    }
    double tot[1];
    if (grid_sum<1, NT>(acc, tot, ws, 0) && threadIdx.x == 0) out[0] = (float)(0.5 * tot[0] / (double)S);
}

// launch geometry of the persistent kernel: SM count x resident CTAs per SM for this instantiation / smem size
template <int NC, int WHAT>
static int launch_tile(const PpoArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    constexpr int PPO_R = PPO_CT;
    const PpoTileLayout L = ppo_layout(a.N, a.logit_pre != nullptr, a.weight != nullptr, PPO_R);
    const size_t smem = (size_t)PPO_STAGES * L.stage_bytes + (WHAT != PPO_FWD ? (size_t)PPO_OUTBUFS * L.logit_bytes : 0) +
                        2 * PPO_STAGES * sizeof(uint64_t);
    constexpr auto kern = ppo_tile_kernel<NC, WHAT>;
    if (smem > 227 * 1024) return B200RL_ERR_ARG;
    int sm_count, per_sm;
    if (int rc = resident_ctas<kern>(PPO_THREADS, smem, sm_count, per_sm)) return rc;
    if (per_sm > 6) per_sm = 6;
    const long long n_tiles = (a.S + PPO_R - 1) / PPO_R;
    // the verification launch that follows a fused forward normally exits at once: keep its grid to one CTA per SM
    long long grid = (long long)sm_count * ((WHAT == PPO_BWD && a.rec.used) ? 1 : per_sm);
    if (grid > n_tiles) grid = n_tiles;
    if (WHAT != PPO_BWD && !ws_partials_fit((long long)(grid * 6), ws_bytes)) return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, PPO_THREADS, smem, st, a, out, ws)) return rc;
    if (WHAT == PPO_BWD) return B200RL_OK;
    return launch_finalize(ws, out, ppo_finalize_args(a.S, a.logit_pre != nullptr, (int)grid), st);
}

template <int WHAT>
static int dispatch_tile(const PpoArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    return with_nc(a.N, [&](auto nc) { return launch_tile<nc, WHAT>(a, out, ws, ws_bytes, st); });
}

}  // namespace b200rl

using namespace b200rl;

static int fill_args(PpoArgs& a, const float* logit_new, const float* logit_old, const float* logit_pretrained,
                     const long long* action, const float* value_new, const float* value_old, const float* adv,
                     const float* return_, const float* weight, long long S, long long G, long long N,
                     double clip_ratio, int use_value_clip, double dual_clip, int kl_type, const float* adv_stats,
                     const float* factor) {
    a.adv_stats = adv_stats;
    a.factor = factor;
    a.logit_new = logit_new; a.logit_old = logit_old; a.logit_pre = logit_pretrained; a.action = action;
    a.value_new = value_new; a.value_old = value_old; a.adv = adv; a.ret = return_; a.weight = weight;
    a.S = S; a.G = (int)G; a.N = (int)N; a.clip = (float)clip_ratio; a.clip_lo = (float)(1.0 - clip_ratio);
    a.clip_hi = (float)(1.0 + clip_ratio); a.dual_clip = (float)dual_clip;
    a.use_value_clip = use_value_clip; a.kl_type = kl_type;
    if (S < 0 || G < 1 || N < 1) return B200RL_ERR_ARG;
    if (!logit_new || !logit_old || !action || !value_new || !value_old || !adv || !return_) return B200RL_ERR_ARG;
    if (kl_type < 1 || kl_type > 3) return B200RL_ERR_ARG;
    return B200RL_OK;
}

extern "C" int b200rl_ppo_fwd(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                              const long long* action, const float* value_new, const float* value_old,
                              const float* adv, const float* return_, const float* weight, long long S, long long G,
                              long long N, double clip_ratio, int use_value_clip, double dual_clip, int kl_type,
                              const float* adv_stats, const float* factor, float* out, float* workspace,
                              size_t workspace_bytes, void* stream) {
    PpoArgs a{};
    int rc = fill_args(a, logit_new, logit_old, logit_pretrained, action, value_new, value_old, adv, return_, weight,
                       S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, adv_stats, factor);
    if (rc != B200RL_OK || !out || !workspace) return rc != B200RL_OK ? rc : B200RL_ERR_ARG;
    if (S == 0) return B200RL_ERR_ARG;  // mean over an empty batch is undefined (reference returns nan)
    cudaStream_t st = (cudaStream_t)stream;
    if (tile_path_ok(a)) return dispatch_tile<PPO_FWD>(a, out, workspace, workspace_bytes, st);
    constexpr int NT = 128;
    const bool warp = a.N > 64;
    int grid = warp ? div_up(S, NT / 32) : div_up(S, NT);
    if (grid > NUM_SMS * 16) grid = NUM_SMS * 16;  // grid-stride kernel: the workspace need is bounded whatever S is
    if (!ws_partials_fit((long long)((size_t)grid * 6), workspace_bytes)) return B200RL_ERR_WORKSPACE;
    if (warp) return launch_k(ppo_fwd_kernel<NT, 2>, grid, NT, 0, st, a, out, workspace);
    return launch_k(ppo_fwd_kernel<NT, 1>, grid, NT, 0, st, a, out, workspace);
}

extern "C" int b200rl_ppo_fwd_grad(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                                   const long long* action, const float* value_new, const float* value_old,
                                   const float* adv, const float* return_, const float* weight, long long S,
                                   long long G, long long N, double clip_ratio, int use_value_clip, double dual_clip,
                                   int kl_type, const float* adv_stats, const float* factor, const float* g_expected,
                                   float* g_used, float* out,
                                   float* grad_logit_new, float* grad_value_new, float* workspace,
                                   size_t workspace_bytes, void* stream) {
    PpoArgs a{};
    int rc = fill_args(a, logit_new, logit_old, logit_pretrained, action, value_new, value_old, adv, return_, weight,
                       S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, adv_stats, factor);
    if (rc != B200RL_OK) return rc;
    if (!workspace || S == 0 || !upstream_args_ok(0, out, true, grad_logit_new && grad_value_new, g_expected, g_used))
        return B200RL_ERR_ARG;
    a.rec = forward_record(g_expected, g_used); a.grad_logit = grad_logit_new; a.grad_value = grad_value_new;
    if (!tile_path_ok(a)) return B200RL_ERR_ARG;  // callers probe with b200rl_ppo_fused_supported first
    return dispatch_tile<PPO_FWD_GRAD>(a, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int b200rl_ppo_fused_supported(const float* logit_new, const float* logit_old,
                                          const float* logit_pretrained, const long long* action,
                                          const float* value_new, const float* value_old, const float* adv,
                                          const float* return_, const float* weight, const float* grad_logit_new,
                                          long long G, long long N) {
    PpoArgs a{};
    a.logit_new = logit_new; a.logit_old = logit_old; a.logit_pre = logit_pretrained; a.action = action;
    a.value_new = value_new; a.value_old = value_old; a.adv = adv; a.ret = return_; a.weight = weight;
    a.grad_logit = const_cast<float*>(grad_logit_new); a.G = (int)G; a.N = (int)N;
    return tile_path_ok(a) ? 1 : 0;
}

extern "C" int b200rl_ppo_bwd(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                              const long long* action, const float* value_new, const float* value_old,
                              const float* adv, const float* return_, const float* weight, long long S, long long G,
                              long long N, double clip_ratio, int use_value_clip, double dual_clip, int kl_type,
                              const float* adv_stats, const float* factor, const float* g_policy, const float* g_value,
                              const float* g_entropy, const float* g_kl,
                              const float* g_used, float* g_hint, float* grad_logit_new, float* grad_value_new,
                              void* stream) {
    PpoArgs a{};
    int rc = fill_args(a, logit_new, logit_old, logit_pretrained, action, value_new, value_old, adv, return_, weight,
                       S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, adv_stats, factor);
    if (rc != B200RL_OK) return rc;
    if (!upstream_args_ok(1, nullptr, true, grad_logit_new && grad_value_new, nullptr, g_used)) return B200RL_ERR_ARG;
    a.rec = verify_record(g_policy, g_value, g_entropy, g_kl, g_used, g_hint);
    a.grad_logit = grad_logit_new; a.grad_value = grad_value_new;
    if (S == 0) return B200RL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int NT = 128;
    if (tile_path_ok(a)) {
        // the check of a learner step: it extends the step chain it follows (common.cuh) by what it may write
        const ChainPoint at = capture_now(st);
        if (int rc = dispatch_tile<PPO_BWD>(a, nullptr, nullptr, 0, st)) return rc;
        const ByteSpan w[] = {byte_span(grad_logit_new, S * G * N * 4), byte_span(grad_value_new, S * 4),
                              byte_span(g_hint, 4 * sizeof(float))};
        chain_report(st, at, false, w, 3);
        return B200RL_OK;
    }
    if (g_used) return B200RL_ERR_ARG;  // the fused forward only exists on the tile path
    long long grid = a.N > 64 ? div_up(S, NT / 32) : div_up(S, NT);
    if (grid > NUM_SMS * 32) grid = NUM_SMS * 32;  // grid-stride kernels
    if (a.N > 64) return launch_k(ppo_bwd_kernel<NT, 2>, (int)grid, NT, 0, st, a);
    return launch_k(ppo_bwd_kernel<NT, 1>, (int)grid, NT, 0, st, a);
}

extern "C" int b200rl_ppo_value_fwd(const float* value_new, const float* value_old, const float* return_,
                                    const float* weight, long long S, double clip_ratio, int use_value_clip,
                                    float* loss, float* dvalue_unit, float* workspace, size_t workspace_bytes,
                                    void* stream) {
    if (!value_new || !return_ || (use_value_clip && !value_old) || !loss || !workspace || S < 1) return B200RL_ERR_ARG;
    constexpr int NT = 256;
    long long grid = div_up(S, NT);
    if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
    if (workspace_bytes < WS_MIN_BYTES || !ws_partials_fit((long long)(grid), workspace_bytes))
        return B200RL_ERR_WORKSPACE;
    return launch_k(ppo_value_kernel<NT>, (int)grid, NT, 0, (cudaStream_t)stream, value_new, value_old, return_, weight,
                    S, (float)clip_ratio, use_value_clip, loss, dvalue_unit, workspace);
}
