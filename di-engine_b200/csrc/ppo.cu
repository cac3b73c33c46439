// PPO clipped surrogate + value + entropy (+ optional KL-to-pretrained) loss, forward and backward.
// Replaces ppo_error / ppo_policy_error / ppo_value_error of ding/rl_utils/ppo.py:77-275 (~40 torch kernels forward
// plus the autograd backward, and two .item() host syncs).
//
// Shapes: S samples, G "agent" rows per sample (G == 1 except the multi-agent case ppo.py:199-200,206-207),
// N logits per row.  logit_* are (S*G, N) row-major, action (S*G) int64, value_new/value_old/adv/return_/weight (S).
//
// Main path (G == 1, N <= 32, 16-byte aligned tensors): ppo_tile_kernel
//   * one CTA per SM (at most), each owning one contiguous span of 256-row tiles (spans differ by at most one tile; only
//     the grid's last tile may be ragged), geometry picked on the host by ps_pick;
//   * every input of a tile -- the logit rows (256*N contiguous floats per tensor), the int64 actions and the four
//     per-sample scalars -- arrives in shared memory by TMA 1-D bulk copies (cp.async.bulk, SASS UBLKCP) that complete
//     on an mbarrier; the ring is as deep as shared memory allows (8 stages at N = 6), and the producer keeps at most
//     PS_AHEAD = 2 stages in flight;
//   * thread i of the 8 consumer warps owns row i of the tile; N is a template parameter (rows live in registers, loops
//     fully unrolled) and the softmax statistics use ex2/lg2 approximations (relative error ~1e-7, far inside the 1e-5
//     parity bar);
//   * a gradient row replaces the row's logit_new slot in the stage; each warp's 32 rows leave as one TMA bulk store
//     (cp.async.bulk.global.shared::cta) and the stage is released once the store has read it;
//   * loss partial sums stay in registers across tiles; one deterministic grid reduction per CTA at the end.
//   Why this geometry: the previous one (128-row tiles, 6 CTAs of 4 consumer warps per SM, a 3-stage ring each, tiles
//   dealt round-robin) put about 22 MB in flight before any tile landed and gave a CTA about 5 tiles, so the ring barely
//   reached steady state.  Measured at config P (S = 524 288, N = 6) on an H100 SXM (700 W, SM clock 1980 MHz):
//   * bench.py: step 47.07 - 47.11 us -> 40.47 us (three runs each); the ppo_fwd_grad call alone (kernel + finalize,
//     back to back over rotated sets) 24.2 -> 23.9 us, 2.28 TB/s on 104 B per transition.  The step gains far more than
//     the call: the old step was 6.3 us longer than its three calls timed alone, the new one is not.  Likely cause (not
//     measured): with PDL the PPO launch is resident while gae_returns still runs, and six old CTAs per SM held 960
//     threads and about 61 K of the 64 K registers there; one new CTA holds 288 threads and 21 K registers.
//   * tools/trace_ppo.py: a CTA's first stage lands 2.8 us (median) after its griddepcontrol.wait, then one stage every
//     1.04 us and the CTA ends 1.0 us after its last stage; 21 - 23 us from the first wait to the last CTA's end.  The
//     per-stage pace is 3.4 TB/s of the 104 B, more than HBM delivers; presumably (not measured) the gradient stores drain
//     into L2 behind the loads, and adv, value and return, written by gae_returns just before, partly come from L2.
//   Slower, not kept: a ring of at most 4 stages (42.55 - 42.59 us per config P step), 128-row stages with 4 consumer
//   warps (63.35 - 63.42 us); no change: 3 stages in flight instead of 2 (40.34 - 40.44 us against 40.39 - 40.42).
//   Not built: starting the loads before griddepcontrol.wait when the kernel follows gae_returns in a captured step.
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

// Geometry of ppo_tile_kernel (its own: fused.cu and pg.cu keep the PPO_* constants of ppo_math.cuh)
constexpr int PS_CW = 8;                  // consumer warps
constexpr int PS_R = PS_CW * 32;          // rows per stage, one per consumer thread
constexpr int PS_THREADS = PS_R + 32;     // + the producer warp
constexpr int PS_MAX_STAGES = 8;          // ring depth where shared memory allows
constexpr int PS_AHEAD = 2;               // stages the producer keeps in flight
constexpr size_t PS_SMEM_LIMIT = 227 * 1024 - 1024;  // dynamic shared memory of one CTA per SM (static partial sums aside)
// B200RL_FUSED_TRACE=1: %globaltimer stamps, 64 per CTA at workspace word 65536 (tools/trace_ppo.py).  0 start, 1 the
// previous launches' results visible (griddepcontrol.wait returned), 2 first stage landed, 3 last stage landed, 4 end
// (partial sums stored), 5 stages of the CTA (low 32 bits) and its SM (high 32 bits); 8 + j stage j landed (j < 56).
constexpr int PS_TRACE_STAGES = 56;

template <int NC, int WHAT>
__global__ void __launch_bounds__(PS_THREADS, 1) ppo_tile_kernel(PpoArgs a, float* ws, int n_stages, int trace) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned long long* tr = trace ? reinterpret_cast<unsigned long long*>(ws + 65536) + blockIdx.x * 64 : nullptr;
    if (tr && threadIdx.x == 0) tr[0] = gtimer();
    pdl_prologue();
    if (tr && threadIdx.x == 0) tr[1] = gtimer();
    constexpr bool GRADS = (WHAT != PPO_FWD);
    constexpr bool LOSSES = (WHAT != PPO_BWD);
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x;
    const int wid = tid >> 5, lane = tid & 31;
    const bool has_pre = a.logit_pre != nullptr, has_w = a.weight != nullptr;
    const PpoTileLayout L = ppo_layout(N, has_pre, has_w, PS_R);
    const int NS = n_stages;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + NS * L.stage_bytes);
    uint64_t* empty = full + PS_MAX_STAGES;

    float g[4] = {0.f, 0.f, 0.f, 0.f};
    // BWD: returns when the forward pass wrote exactly these gradients
    if (GRADS && upstream<4>(a.rec, WHAT == PPO_BWD, ppo_owned(a), g)) return;
    const PpoUpstream up{g[0], g[1], g[2], g[3], 1.f / (float)a.S};

    // CTA b owns the contiguous tiles [t0, t1): spans differ by at most one tile, and only the grid's last tile may be
    // ragged.  A static map, so the per-CTA partial sums (and with them the losses) do not depend on timing.
    const long long n_full = a.S / PS_R;
    const int tail_rows = (int)(a.S - n_full * PS_R);
    const long long n_tiles = n_full + (tail_rows ? 1 : 0);
    const long long t0 = n_tiles * blockIdx.x / gridDim.x, t1 = n_tiles * (blockIdx.x + 1) / gridDim.x;
    const int my_n = (int)(t1 - t0);

    if (tid == 0) {
        for (int s = 0; s < NS; ++s) {
            mbar_init(&full[s], 1);        // producer's expect_tx arrive + TMA byte count
            mbar_init(&empty[s], PS_CW);   // one arrive per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // policy, value, entropy, kl, approx_kl, clipfrac
    if (wid == PS_CW) {
        // ---- producer: one lane issues every stage's bulk copies, at most PS_AHEAD stages in flight --------------------
        if (lane == 0) {
            for (int i = 0; i < my_n; ++i) {
                const long long t = t0 + i;
                if (t >= n_full) break;  // the ragged last tile is read with plain loads by its consumers
                const int sg = i % NS;
                if (i >= NS) mbar_wait(&empty[sg], (uint32_t)(((i / NS) - 1) & 1));
                if (NS > PS_AHEAD && i >= PS_AHEAD) {  // stage i - PS_AHEAD has landed
                    const int jb = i - PS_AHEAD;
                    mbar_wait(&full[jb % NS], (uint32_t)((jb / NS) & 1));
                }
                const long long row0 = t * PS_R;
                unsigned char* st = smem + sg * L.stage_bytes;
                uint64_t* bar = &full[sg];
                mbar_expect_tx(bar, (uint32_t)L.tx_bytes);
                tma_load_1d(st, a.logit_new + row0 * N, L.logit_bytes, bar);
                tma_load_1d(st + L.off_old, a.logit_old + row0 * N, L.logit_bytes, bar);
                if (has_pre) tma_load_1d(st + L.off_pre, a.logit_pre + row0 * N, L.logit_bytes, bar);
                tma_load_1d(st + L.off_act, a.action + row0, PS_R * 8, bar);
                tma_load_1d(st + L.off_vn, a.value_new + row0, PS_R * 4, bar);
                tma_load_1d(st + L.off_vo, a.value_old + row0, PS_R * 4, bar);
                tma_load_1d(st + L.off_adv, a.adv + row0, PS_R * 4, bar);
                tma_load_1d(st + L.off_ret, a.ret + row0, PS_R * 4, bar);
                if (has_w) tma_load_1d(st + L.off_w, a.weight + row0, PS_R * 4, bar);
            }
        }
    } else {
        // ---- consumers: warp w owns rows [32w, 32w+32) of every stage; no CTA-wide barrier in this loop ----------------
        const int rit = wid * 32 + lane;  // this thread's row in every stage
        const int warp_out_bytes = 32 * N * 4;
        for (int i = 0; i < my_n; ++i) {
            const long long t = t0 + i;
            const long long row0 = t * PS_R;
            const int sg = i % NS;
            unsigned char* st = smem + sg * L.stage_bytes;
            const bool full_tile = t < n_full;
            if (full_tile) {
                mbar_wait(&full[sg], (uint32_t)((i / NS) & 1));
                if (tr && tid == 0) {
                    const unsigned long long now = gtimer();
                    if (i == 0) tr[2] = now;
                    tr[3] = now;
                    if (i < PS_TRACE_STAGES) tr[8 + i] = now;
                }
            } else if (rit < tail_rows) {
                // ragged last tile: every thread fetches its own row into its own slots of the stage (no sharing); the
                // bulk stores that read this slot earlier have finished reading it (wait_read + __syncwarp below)
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
            // a full stage's gradient rows replace the rows' own logit_new slots (ppo_row_compute_to reads them first)
            if (full_tile || rit < tail_rows) {
                const float adv = reinterpret_cast<const float*>(st + L.off_adv)[rit];
                ppo_row_compute<NC, LOSSES, GRADS>(a, L, st, rit, N, adv, full_tile, reinterpret_cast<float*>(st), row0,
                                                   up, acc);
            }
            if (!full_tile) continue;
            if (GRADS) {
                // this warp's 32 gradient rows are one contiguous span: one bulk store.  The stage is released once the
                // store has read it -- with a ring of two or more, one stage later, so the warp does not wait for it
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                    tma_store_1d(a.grad_logit + (row0 + wid * 32) * N, st + wid * warp_out_bytes, warp_out_bytes);
                    tma_store_commit();
                    if (NS == 1) {
                        tma_store_wait_read<0>();
                        mbar_arrive(&empty[sg]);
                    } else {
                        tma_store_wait_read<1>();
                        if (i > 0) mbar_arrive(&empty[(i - 1) % NS]);
                    }
                }
                // only lane 0 waited for the store's read: the other lanes may write this warp's rows of the ring again
                // (the ragged last tile's plain loads) only after it
                __syncwarp();
            } else {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[sg]);  // stage may be refilled once all consumer warps have arrived
            }
        }
        if (GRADS && lane == 0) tma_store_wait_read<0>();  // shared memory must outlive the bulk stores that read it
    }
    if (LOSSES) grid_store_partials<6, PS_THREADS>(acc, ws);  // summed by finalize_sums_kernel, launched right behind
    if (tr && tid == 0) {
        tr[4] = gtimer();
        tr[5] = (unsigned long long)smid() << 32 | (unsigned long long)my_n;
    }
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

// Geometry for S rows of N logits on `sm_count` SMs (one CTA per SM at most): the grid, the ring depth and the dynamic
// shared memory.  The ring is as deep as shared memory allows, up to PS_MAX_STAGES and no deeper than a CTA has tiles
// (small batches, e.g. PPO minibatches of 64 - 320 rows, get one or two CTAs and a short ring).  The verification launch
// behind a fused forward normally returns at once: it gets one stage, so that it holds little shared memory while the
// next step's kernel starts beside it, and recomputes on that one stage when the record says so.  At config D (N = 6)
// that launch holds 18.5 KB of shared memory, 288 threads and 288 x 72 = 20.7 K registers per SM (ptxas, sm_90a); the
// column kernel of the next step (gae_ppo_ws_kernel<6, true, 32>) needs about 165 KB, 320 threads and 320 x 96 = 30.7 K
// registers, so both fit on one SM at once.
struct PsGeo {
    int grid, stages;
    size_t smem;
};
static PsGeo ps_pick(long long S, int N, bool has_pre, bool has_w, bool verify_only, int sm_count) {
    PsGeo g{};
    const size_t stage = (size_t)ppo_layout(N, has_pre, has_w, PS_R).stage_bytes;
    const size_t bars = 2 * PS_MAX_STAGES * sizeof(uint64_t);
    const long long n_tiles = (S + PS_R - 1) / PS_R;
    g.grid = (int)(n_tiles < sm_count ? n_tiles : sm_count);
    const long long per_cta = g.grid > 0 ? (n_tiles + g.grid - 1) / g.grid : 0;
    long long stages = verify_only ? 1 : (long long)((PS_SMEM_LIMIT - bars) / stage);
    if (stages > PS_MAX_STAGES) stages = PS_MAX_STAGES;
    if (stages > per_cta) stages = per_cta;
    g.stages = stages < 1 ? 0 : (int)stages;  // 0: not even one stage fits
    g.smem = (size_t)g.stages * stage + bars;
    return g;
}

template <int NC, int WHAT>
static int launch_tile(const PpoArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    int sm_count = 0;
    if (int rc = sm_count_of(sm_count)) return rc;
    const PsGeo g = ps_pick(a.S, a.N, a.logit_pre != nullptr, a.weight != nullptr, WHAT == PPO_BWD && a.rec.used, sm_count);
    if (g.stages < 1) return B200RL_ERR_ARG;
    constexpr auto kern = ppo_tile_kernel<NC, WHAT>;
    if (int rc = smem_opt_in<kern>(g.smem)) return rc;
    if (WHAT != PPO_BWD && !ws_partials_fit((long long)g.grid * 6, ws_bytes)) return B200RL_ERR_WORKSPACE;
    const int trace = WHAT != PPO_BWD && trace_enabled();
    if (trace && (size_t)65536 * 4 + (size_t)g.grid * 64 * 8 > ws_bytes) return B200RL_ERR_WORKSPACE;  // the stamps
    if (int rc = launch_k(kern, g.grid, PS_THREADS, g.smem, st, a, ws, g.stages, trace)) return rc;
    if (WHAT == PPO_BWD) return B200RL_OK;
    return launch_finalize(ws, out, ppo_finalize_args(a.S, a.logit_pre != nullptr, g.grid), st);
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

extern "C" int b200rl_ppo_tile_geometry(long long S, long long N, int has_pretrained, int has_weight, int verify_only,
                                        int sm_count, long long* geometry3) {
    if (S < 1 || N < 1 || N > 32 || sm_count < 1 || !geometry3) return B200RL_ERR_ARG;
    const PsGeo g = ps_pick(S, (int)N, has_pretrained != 0, has_weight != 0, verify_only != 0, sm_count);
    geometry3[0] = g.grid; geometry3[1] = g.stages; geometry3[2] = (long long)g.smem;
    return B200RL_OK;
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
