// V-trace learner step in ONE launch: vtrace_error_discrete_action forward AND the gradients w.r.t. target_output and value
// (ding/rl_utils/vtrace.py:72-136, isw.py:55-58), column tiles, warp-specialised -- the scheme of colws.cu applied to the
// IMPALA loss.  The batch crosses HBM once: 68 B read + 28 B written per transition (N = 6) instead of the ~150 B that the
// three launches of pg.cu (rows -> scan -> backward tiles) move.
//
// A CTA owns TC = 16 batch columns for ALL T (the recurrences run along T only).  Time is walked newest-first in chunks of
// R = 16 steps (256 transitions, thread = transition).  Per chunk three parties hand work to each other through mbarriers:
//   consumers, phase A   softmax statistics of the target row (logsumexp, entropy) and of the behaviour row, log pi(a),
//                        importance weight IS = exp(log pi(a) - log mu(a)) (isw.py:55-58) -> shared memory
//   scanner              delta_t = min(IS, rho) (r_t + g V_{t+1} - V_t), x_t = delta_t + g*l*min(IS, c) x_{t+1},
//                        vs_t = V_t + x_t (vtrace.py:22-29) -> shared memory, together with vs of the row above the chunk
//   consumers, phase B   adv_t = min(IS, rho_pg) (r_t + g vs_{t+1} - V_t) (vtrace.py:126-128), the three loss terms
//                        (:130-135), the gradient row of target_output and d loss / d V_t, stored straight to HBM
// The consumers run phase A one chunk ahead of phase B (A(j+1) while the scanner works on chunk j), a loader warp keeps an
// S-stage ring of target logits | behaviour logits | actions [| weights] full with 16-byte cp.async copies, and the scanner
// fetches its own value / reward rows two chunks ahead.
//
// Backward contract (as ppo.cu's FWD_GRAD): the gradients are produced in the forward launch for the upstream gradients the
// training loop is expected to send (g_expected, remembered on the device).  backward() launches the same kernel in verify
// mode: every CTA compares the actual upstream gradients with the recorded ones (upstream(), common.cuh) and exits at once
// when they agree; otherwise the whole step is recomputed with the actual values.  Exact for any upstream gradient, no host
// sync.
#include "../../include/b200rl.h"
#include "ppo_math.cuh"

namespace b200rl {

constexpr int VW_CW = 8;
constexpr int VW_CT = VW_CW * 32;        // consumer threads = transitions per chunk
constexpr int VW_THREADS = VW_CT + 32 + 32;  // consumers + loader warp + scanner warp
constexpr int VW_MAX_STAGES = 4;
// tile width TC (template parameter): 16 columns x 16 time steps per chunk, or 32 x 8 when 16-column tiles would outnumber
// the resident CTAs (two per SM): a second wave of 16-column tiles leaves the second half of the kernel under-subscribed,
// while 32-column tiles all stream from start to end

struct VtFusedArgs {
    const float* target;      // (T*B, N)
    const float* behaviour;   // (T*B, N)
    const long long* action;  // (T*B)
    const float* value;       // (T+1, B)
    const float* reward;      // (T, B)
    const float* weight;      // nullable (T, B)
    long long T, B;
    int N;
    float gamma, gamma_lambda, rho_clip, c_clip, rho_pg_clip;
    UpstreamRecord rec;       // slots policy, value, entropy
    float* grad_logit;        // (T*B, N), nullable = losses only
    float* grad_value;        // (T+1, B)
    int trace;
};

// timeline instrumentation (B200RL_FUSED_TRACE=1, tools/trace_vt.py): 64 globaltimer stamps per CTA at workspace word 65536;
// chunk j < 8: consumers 4j (A: stage landed), 4j+1 (A done), 4j+2 (B: vs ready), 4j+3 (B done);
// scanner 32+2j (IS ready), 33+2j (vs published); loader 48+2j (stage free), 49+2j (copies issued)
#define VW_TRACE(slot)                                                                                       \
    do {                                                                                                     \
        if (a.trace) reinterpret_cast<unsigned long long*>(ws + 65536)[blockIdx.x * 64 + (slot)] = gtimer(); \
    } while (0)

struct VwItem {
    long long tile;
    long long q;  // chunk from the top: time steps [T - (q+1)R, T - qR)
};

__host__ __device__ inline int vw_stage_bytes(int N, bool has_w, int tc) {
    // logits x2 | action | [weight] | value rows (R+1) | reward rows | IS | vs rows (R+1);  R * tc == VW_CT
    const int row = tc * 4;
    return VW_CT * (2 * N * 4 + 8 + (has_w ? 4 : 0)) + (VW_CT * 4 + row) + VW_CT * 4 + VW_CT * 4 + (VW_CT * 4 + row);
}

template <int NC, bool GRADS, int TC>
__global__ void __launch_bounds__(VW_THREADS, 2) vtrace_ws_kernel(VtFusedArgs a, float* ws, int S) {
    constexpr int VW_TC = TC;             // columns per tile
    constexpr int VW_R = VW_CT / VW_TC;   // time steps per chunk
    constexpr int VW_ROW = VW_TC * 4;     // bytes of one (T, B) row segment of the tile
    constexpr int PPR = VW_TC / 4;        // 16-byte pieces per (T, B) row segment
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ __align__(128) unsigned char smem[];
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const bool has_w = a.weight != nullptr;
    // stage layout
    const int lb = VW_CT * N * 4;
    const int off_beh = lb, off_act = 2 * lb, off_w = off_act + VW_CT * 8;
    const int off_v = off_w + (has_w ? VW_CT * 4 : 0);     // [R+1][TC] value rows t0 .. t0+R
    const int off_r = off_v + (VW_R + 1) * VW_ROW;         // [R][TC] reward
    const int off_is = off_r + VW_R * VW_ROW;              // [R][TC] importance weights (phase A -> scanner, phase B)
    const int off_vs = off_is + VW_CT * 4;                 // [R+1][TC] vs rows (row R = the row above the chunk)
    const int stage_bytes = off_vs + (VW_R + 1) * VW_ROW;  // multiple of 64
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * stage_bytes);
    uint64_t* full = bars;                           // [S] stage landed (32 loader-lane arrivals)
    uint64_t* is_ready = bars + VW_MAX_STAGES;       // [S] phase A done (VW_CW arrivals)
    uint64_t* vs_ready = bars + 2 * VW_MAX_STAGES;   // [S] scanner done (1 arrival)
    uint64_t* done = bars + 3 * VW_MAX_STAGES;       // [S] phase B done: stage free (VW_CW arrivals)

    const long long T = a.T, B = a.B;
    const long long n_tiles = (B + VW_TC - 1) / VW_TC;
    const long long n_chunks = (T + VW_R - 1) / VW_R;

    if (tid == 0) {
        for (int s = 0; s < VW_MAX_STAGES; ++s) {
            mbar_init(&full[s], 32);
            mbar_init(&is_ready[s], VW_CW);
            mbar_init(&vs_ready[s], 1);
            mbar_init(&done[s], VW_CW);
        }
        mbar_fence_init();
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float g[3] = {0.f, 0.f, 0.f};
    if (GRADS && upstream<3>(a.rec, a.rec.verify, 7u, g)) return;  // uniform over the grid
    const float g_pg = g[0], g_val = g[1], g_ent = g[2];
    __syncthreads();

    auto item_valid = [&](const VwItem& it) { return it.tile < n_tiles; };
    auto item_next = [&](VwItem& it) {
        if (++it.q >= n_chunks) {
            it.q = 0;
            it.tile += gridDim.x;
        }
    };
    const VwItem first{(long long)blockIdx.x, 0};
    float acc[3] = {0.f, 0.f, 0.f};

    if (wid == VW_CW) {
        // =============================================== loader ===========================================================
        auto rows_of = [&](unsigned char* dst, const void* src, long long t0, long long c0, int esz, int jmin, int W) {
            const int P = VW_TC * esz / 16, Pv = W * esz / 16;
            const unsigned char* g = reinterpret_cast<const unsigned char*>(src) + (t0 * B + c0) * esz;
            const long long rstride = B * esz;
            const int n = VW_R * P;
#pragma unroll 4
            for (int p = lane; p < n; p += 32) {
                const int row = p / P, o = p - row * P;
                if (row >= jmin && o < Pv) cpa16(dst + p * 16, g + row * rstride + o * 16);
            }
        };
        // (loop-invariant piece offsets in registers, as tried in colws.cu, are slower here too)
        VwItem it = first;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            if (j >= S) mbar_wait(&done[s], (uint32_t)(ph ^ 1));
            if (tid == VW_CT && j < 8) VW_TRACE(48 + 2 * j);
            const long long c0 = it.tile * VW_TC;
            const long long t0 = T - (it.q + 1) * VW_R;
            const int jmin = t0 < 0 ? (int)-t0 : 0;
            const int W = (int)((B - c0) < VW_TC ? (B - c0) : VW_TC);
            unsigned char* st = smem + s * stage_bytes;
            if (jmin == 0 && W == VW_TC) {
                // full chunk of a full tile: lane-owns-a-piece-column copies (common.cuh warp_copy_rows); a row segment is
                // TC * esz / 16 pieces = (TC / 4) * (N | 2 | 1) for logits | actions | weights
                const uint32_t sb = smem_u32(st);
                const long long e0 = t0 * B + c0;
                warp_copy_rows<VW_TC / 4, VW_R, NC>(sb, a.target + e0 * N, B * N * 4, N, lane);
                warp_copy_rows<VW_TC / 4, VW_R, NC>(sb + off_beh, a.behaviour + e0 * N, B * N * 4, N, lane);
                warp_copy_rows<VW_TC / 4, VW_R, 2>(sb + off_act, a.action + e0, B * 8, 2, lane);
                if (has_w) warp_copy_rows<VW_TC / 4, VW_R, 1>(sb + off_w, a.weight + e0, B * 4, 1, lane);
            } else {
                rows_of(st, a.target, t0, c0, N * 4, jmin, W);
                rows_of(st + off_beh, a.behaviour, t0, c0, N * 4, jmin, W);
                rows_of(st + off_act, a.action, t0, c0, 8, jmin, W);
                if (has_w) rows_of(st + off_w, a.weight, t0, c0, 4, jmin, W);
            }
            cpa_mbar_arrive(&full[s]);
            if (tid == VW_CT && j < 8) VW_TRACE(49 + 2 * j);
            if (++s == S) { s = 0; ph ^= 1; }
            item_next(it);
        }
    } else if (wid == VW_CW + 1) {
        // =============================================== scanner ==========================================================
        // value rows t0 .. t0+R (R+1 rows: the bootstrap row T belongs to the newest chunk) and reward rows t0 .. t0+R-1 of
        // chunk k go to stage k % S; TC/4 16-byte pieces per row and tensor
        auto issue_raw = [&](const VwItem& it, int sg) {
            const long long c0 = it.tile * VW_TC;
            const long long t0 = T - (it.q + 1) * VW_R;
            const int W = (int)((B - c0) < VW_TC ? (B - c0) : VW_TC);
            unsigned char* st = smem + sg * stage_bytes;
            for (int p = lane; p < (VW_R + 1) * PPR; p += 32) {
                const int row = p / PPR, o = p % PPR;
                if (t0 + row >= 0 && o * 4 < W) cpa16(st + off_v + p * 16, a.value + (t0 + row) * B + c0 + o * 4);
            }
            for (int p = lane; p < VW_R * PPR; p += 32) {
                const int row = p / PPR, o = p % PPR;
                if (t0 + row >= 0 && o * 4 < W) cpa16(st + off_r + p * 16, a.reward + (t0 + row) * B + c0 + o * 4);
            }
        };
        VwItem it = first, pf = first;
        for (int k = 0; k < S; ++k) {  // chunks 0 .. S-1: every stage is free at the start
            if (item_valid(pf)) {
                issue_raw(pf, k);
                item_next(pf);
            }
            cpa_commit();
        }
        float carry = 0.f, above = 0.f;
        int s = 0, ph = 0;
        int s2 = S - 2;  // stage of chunk j-2 == stage of chunk j+S-2
        for (int j = 0; item_valid(it); ++j) {
            const long long c0 = it.tile * VW_TC;
            const long long t0 = T - (it.q + 1) * VW_R;
            unsigned char* st = smem + s * stage_bytes;
            // one cp.async group per prologue chunk and per iteration: chunk j is group j (j < S) or j + 2, of the S + j committed
            // so far -- S - 1 younger groups may stay in flight for the prologue chunks, S - 3 afterwards.  (Waiting for all but
            // one from the first chunk on -- as this line did -- held chunk 0's scan until the rows of chunks 1 and 2 had landed
            // behind the loader's first burst, which delays the first published chunk -- tools/trace_vt_warps.py shows it.)
            if (S >= 4) {
                if (j < S) cpa_wait<3>(); else cpa_wait<1>();
            } else {
                if (j < S) cpa_wait<2>(); else cpa_wait<0>();
            }
            __syncwarp();
            mbar_wait(&is_ready[s], (uint32_t)ph);
            if (lane == 0 && j < 8) VW_TRACE(32 + 2 * j);
            // phase A of chunk j is complete in every consumer warp => phase B of chunk j-2 is, too: its stage is free
            if (j >= 2 && item_valid(pf)) {
                issue_raw(pf, s2);
                item_next(pf);
            }
            cpa_commit();
            const float* sv = reinterpret_cast<const float*>(st + off_v);
            const float* sr = reinterpret_cast<const float*>(st + off_r);
            const float* sis = reinterpret_cast<const float*>(st + off_is);
            float* svs = reinterpret_cast<float*>(st + off_vs);
            if (it.q == 0) {  // newest chunk of a tile: x_T = 0, vs_T = V_T (vtrace.py:24,127); d loss / d V_T = 0
                carry = 0.f;
                above = (lane < VW_TC && c0 + lane < B) ? sv[VW_R * VW_TC + lane] : 0.f;
                if (GRADS && lane < VW_TC && c0 + lane < B) a.grad_value[T * B + c0 + lane] = 0.f;
            }
            // lane = column: everything the recurrence needs goes to registers first (the shared-memory loads are independent
            // of the carry), then the dependent chain runs on registers only
            if (lane < VW_TC) {
                svs[VW_R * VW_TC + lane] = above;
                if (c0 + lane < B) {
                    if (t0 >= 0) {
                        float d[VW_R], g[VW_R], vv[VW_R + 1];
#pragma unroll
                        for (int k = 0; k <= VW_R; ++k) vv[k] = sv[k * VW_TC + lane];
#pragma unroll
                        for (int k = 0; k < VW_R; ++k) {
                            const float is = sis[k * VW_TC + lane], rw = sr[k * VW_TC + lane];
                            d[k] = fmul(fminf(is, a.rho_clip), fsub(fadd(rw, fmul(a.gamma, vv[k + 1])), vv[k]));
                            g[k] = fmul(a.gamma_lambda, fminf(is, a.c_clip));
                        }
                        float vs = above;
#pragma unroll
                        for (int k = VW_R - 1; k >= 0; --k) {
                            carry = fadd(d[k], fmul(g[k], carry));
                            vs = fadd(vv[k], carry);
                            vv[k] = vs;
                        }
#pragma unroll
                        for (int k = 0; k < VW_R; ++k) svs[k * VW_TC + lane] = vv[k];
                        above = vv[0];
                    } else {  // ragged oldest chunk
                        float vs = above;
                        for (int jj = VW_R - 1; jj >= 0 && t0 + jj >= 0; --jj) {
                            const int e = jj * VW_TC + lane;
                            const float is = sis[e], v = sv[e];
                            const float dl = fmul(fminf(is, a.rho_clip), fsub(fadd(sr[e], fmul(a.gamma, sv[e + VW_TC])), v));
                            carry = fadd(dl, fmul(fmul(a.gamma_lambda, fminf(is, a.c_clip)), carry));
                            vs = fadd(v, carry);
                            svs[e] = vs;
                        }
                        above = vs;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&vs_ready[s]);
                if (j < 8) VW_TRACE(33 + 2 * j);
            }
            if (++s == S) { s = 0; ph ^= 1; }
            if (++s2 == S) s2 = 0;
            item_next(it);
        }
        cpa_wait<0>();
    } else {
        // =============================================== consumers ========================================================
        const float inv_m = 1.f / (float)(T * B);
        const int jj = tid / VW_TC, c = tid % VW_TC;
        constexpr int NR = NC ? NC : 1;
        // state of the chunk whose phase B is pending
        bool pend = false;
        int p_s = 0, p_ph = 0;
        long long p_c0 = 0, p_t = 0;
        float p_lse = 0.f, p_lp = 0.f, p_ent = 0.f, p_is = 0.f;
        VwItem it = first;
        int s = 0, ph = 0;
        for (int j = 0;; ++j) {  // iteration j: phase A of chunk j, phase B of chunk j-1
            const bool have = item_valid(it);
            if (!have && !pend) break;
            // ---- phase A of the next chunk ------------------------------------------------------------------------------
            int n_s = s, n_ph = ph;
            long long n_c0 = 0, n_t = 0;
            float n_lse = 0.f, n_lp = 0.f, n_ent = 0.f, n_is = 0.f;
            if (have) {
                n_c0 = it.tile * VW_TC;
                n_t = T - (it.q + 1) * VW_R + jj;
                unsigned char* st = smem + s * stage_bytes;
                mbar_wait(&full[s], (uint32_t)ph);
                if (tid == 0 && j < 8) VW_TRACE(4 * j);
                if (n_t >= 0 && n_c0 + c < B) {
                    const float* zt = reinterpret_cast<const float*>(st) + tid * N;
                    const float* zb = reinterpret_cast<const float*>(st + off_beh) + tid * N;
                    const int act = (int)reinterpret_cast<const long long*>(st + off_act)[tid];
                    float m = kF32Min, sum = 0.f, u2 = 0.f, mb = kF32Min, sb = 0.f;
                    if (NC) {
                        float z[NR], zo[NR];
                        load_row<NR>(zt, z);
                        load_row<NR>(zb, zo);
#pragma unroll
                        for (int k = 0; k < NR; ++k) { m = fmaxf(m, z[k]); mb = fmaxf(mb, zo[k]); }
                        const float m2 = m * kLog2e, mb2 = mb * kLog2e;
#pragma unroll
                        for (int k = 0; k < NR; ++k) {
                            const float t = fmaxf(fmaf(z[k], kLog2e, -m2), kF32Min);
                            const float e = ex2f_(t);
                            sum += e;
                            u2 = fmaf(e, t, u2);
                            sb += ex2f_(fmaf(zo[k], kLog2e, -mb2));
                        }
                    } else {
                        for (int k = 0; k < N; ++k) { m = fmaxf(m, zt[k]); mb = fmaxf(mb, zb[k]); }
                        const float m2 = m * kLog2e, mb2 = mb * kLog2e;
                        for (int k = 0; k < N; ++k) {
                            const float t = fmaxf(fmaf(zt[k], kLog2e, -m2), kF32Min);
                            const float e = ex2f_(t);
                            sum += e;
                            u2 = fmaf(e, t, u2);
                            sb += ex2f_(fmaf(zb[k], kLog2e, -mb2));
                        }
                    }
                    const float l2s = lg2f_(sum);
                    n_lse = m + l2s * kLn2;
                    n_ent = (l2s - u2 * rcpf_(sum)) * kLn2;
                    n_lp = zt[act] - n_lse;
                    const float lp_b = (zb[act] - mb) - lg2f_(sb) * kLn2;
                    n_is = ex2f_((n_lp - lp_b) * kLog2e);
                    reinterpret_cast<float*>(st + off_is)[tid] = n_is;
                } else {
                    reinterpret_cast<float*>(st + off_is)[tid] = 0.f;
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&is_ready[s]);
                if (tid == 0 && j < 8) VW_TRACE(4 * j + 1);
                if (++s == S) { s = 0; ph ^= 1; }
                item_next(it);
            }
            // ---- phase B of the pending chunk ---------------------------------------------------------------------------
            if (pend) {
                unsigned char* st = smem + p_s * stage_bytes;
                mbar_wait(&vs_ready[p_s], (uint32_t)p_ph);
                if (tid == 0 && j >= 1 && j < 9) VW_TRACE(4 * (j - 1) + 2);
                if (p_t >= 0 && p_c0 + c < B) {
                    const float* sv = reinterpret_cast<const float*>(st + off_v);
                    const float* svs = reinterpret_cast<const float*>(st + off_vs);
                    const float v = sv[tid], rw = reinterpret_cast<const float*>(st + off_r)[tid];
                    const float w = has_w ? reinterpret_cast<const float*>(st + off_w)[tid] : 1.f;
                    const float adv = fmul(fminf(p_is, a.rho_pg_clip), fsub(fadd(rw, fmul(a.gamma, svs[tid + VW_TC])), v));
                    const float dv = v - svs[tid];
                    acc[0] += p_lp * adv * w;
                    acc[1] += dv * dv * w;
                    acc[2] += p_ent * w;
                    if (GRADS) {
                        const long long g = p_t * B + p_c0 + c;
                        const float* zt = reinterpret_cast<const float*>(st) + tid * N;
                        const int act = (int)reinterpret_cast<const long long*>(st + off_act)[tid];
                        // grad z_j = g_pg (-adv w / M)(1[j==a] - p_j) + g_ent (w / M)(-p_j (log p_j + H))
                        // (log p_j clamped at finfo.min as Categorical.entropy does: p_j = 0 at a -inf logit times a finite number)
                        const float c_act = g_pg * (-adv * w) * inv_m, c_ent = g_ent * w * inv_m;
                        float* gz = a.grad_logit + g * N;
                        if (NC) {
                            float z[NR], gj[NR];
                            load_row<NR>(zt, z);
#pragma unroll
                            for (int k = 0; k < NR; ++k) {
                                const float lpk = fmaxf(z[k] - p_lse, kF32Min);
                                const float p = ex2f_(lpk * kLog2e);
                                gj[k] = -c_act * p - c_ent * p * (lpk + p_ent);
                                if (k == act) gj[k] += c_act;
                            }
                            store_row<NR>(gz, gj);
                        } else {
                            for (int k = 0; k < N; ++k) {
                                const float lpk = fmaxf(zt[k] - p_lse, kF32Min);
                                const float p = ex2f_(lpk * kLog2e);
                                float gk = -c_act * p - c_ent * p * (lpk + p_ent);
                                if (k == act) gk += c_act;
                                gz[k] = gk;
                            }
                        }
                        a.grad_value[g] = g_val * (2.f * w * dv * inv_m);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&done[p_s]);
                if (tid == 0 && j >= 1 && j < 9) VW_TRACE(4 * (j - 1) + 3);
            }
            pend = have;
            p_s = n_s; p_ph = n_ph; p_c0 = n_c0; p_t = n_t;
            p_lse = n_lse; p_lp = n_lp; p_ent = n_ent; p_is = n_is;
        }
    }
    if (!a.rec.verify) grid_store_partials<3, VW_THREADS>(acc, ws);  // summed by finalize_sums_kernel
}

static size_t vw_smem(int N, bool has_w, int stages, int tc) {
    return (size_t)stages * vw_stage_bytes(N, has_w, tc) + 4 * VW_MAX_STAGES * sizeof(uint64_t) + 64;
}
static int vw_pick_stages(int N, bool has_w, int tc = 32) {
    for (int s = VW_MAX_STAGES; s >= 3; --s)
        if (vw_smem(N, has_w, s, tc) <= 112 * 1024) return s;  // two CTAs per SM
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Resident-tile variant for short trajectories (IMPALA unroll lengths: T*TC transitions fit one CTA's shared memory).
// A CTA owns TC columns for all T and loads its WHOLE tile with one burst of 16-byte cp.async copies from all 256 threads
// (every byte of the tile is in flight at once; several CTAs per SM are at different points of load -> phase A -> scan ->
// phase B, so the SM overlaps one tile's arithmetic with its neighbours' loads without any in-CTA pipeline):
//   phase A  (thread = transition, strided)  softmax statistics, IS -> shared; {lse, entropy} parked in the behaviour row,
//                                            which is dead from here on
//   scan     (warp 0, lane = column)         the reverse recurrence in 16-step register batches, vs rows -> shared
//   phase B  (thread = transition)           advantages, the three loss terms, both gradients straight to HBM
// Same arithmetic, operation for operation, as vtrace_ws_kernel; same backward contract (verify launch).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int VR_NT = 256;

__host__ __device__ inline size_t vr_smem_bytes(long long T, int N, bool has_w, int tc) {
    const size_t e = (size_t)T * tc;
    return e * (2 * (size_t)N * 4 + 8 + (has_w ? 4 : 0) + 4 + 4) + 2 * (size_t)(T + 1) * tc * 4 + 16;
}

template <int NC, bool GRADS, int TC>
__global__ void __launch_bounds__(VR_NT) vtrace_res_kernel(VtFusedArgs a, float* ws) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ __align__(128) unsigned char smem[];
    const int N = NC ? NC : a.N;
    constexpr int NR = NC ? NC : 1;
    const int tid = threadIdx.x, lane = tid & 31;
    const bool has_w = a.weight != nullptr;
    const int T = (int)a.T;
    const long long B = a.B;
    const int E = T * TC;  // transitions of the tile, e = t * TC + c
    const long long c0 = (long long)blockIdx.x * TC;
    const int W = (int)((B - c0) < TC ? (B - c0) : TC);
    float* zt = reinterpret_cast<float*>(smem);
    float* zb = zt + (size_t)E * N;
    long long* sact = reinterpret_cast<long long*>(zb + (size_t)E * N);
    float* sw = reinterpret_cast<float*>(sact + E);
    float* sv = sw + (has_w ? E : 0);  // [T+1][TC]
    float* sr = sv + (T + 1) * TC;     // [T][TC]
    float* sis = sr + E;               // [T][TC]
    float* svs = sis + E;              // [T+1][TC]
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float g[3] = {0.f, 0.f, 0.f};
    if (GRADS && upstream<3>(a.rec, a.rec.verify, 7u, g)) return;  // uniform over the grid
    const float g_pg = g[0], g_val = g[1], g_ent = g[2];
    // ---- the whole tile, one burst: per time step one contiguous segment of W * esz bytes per tensor ------------------------
    // A thread owns one 16-byte column of the row segment and walks down the rows: two pointer increments per copy, no
    // division in the loop (the p -> (row, piece) arithmetic of a flat loop was 31 % of the kernel's instructions).
    {
        auto rows = [&](void* dst, const void* src, int n_rows, int esz) {
            const int P = TC * esz / 16, Pv = W * esz / 16;  // pieces per row in shared memory / valid ones
            const long long rstride = B * esz;
            if (P <= VR_NT) {
                const int RP = VR_NT / P;  // rows per pass
                const int r0 = tid / P, o = tid - r0 * P;
                if (r0 < RP && o < Pv) {
                    const unsigned char* g = reinterpret_cast<const unsigned char*>(src) + c0 * esz + r0 * rstride + o * 16;
                    uint32_t d = smem_u32(dst) + (uint32_t)(r0 * P + o) * 16u;
                    const long long gstep = (long long)RP * rstride;
                    const uint32_t dstep = (uint32_t)(RP * P) * 16u;
                    for (int row = r0; row < n_rows; row += RP) {
                        cpa16_s(d, g);
                        g += gstep;
                        d += dstep;
                    }
                }
            } else {  // very wide rows: flat loop
                const unsigned char* g = reinterpret_cast<const unsigned char*>(src) + c0 * esz;
                unsigned char* d = reinterpret_cast<unsigned char*>(dst);
                const int n = n_rows * P;
                for (int p = tid; p < n; p += VR_NT) {
                    const int row = p / P, o = p - row * P;
                    if (o < Pv) cpa16(d + (size_t)p * 16, g + row * rstride + o * 16);
                }
            }
        };
        rows(zt, a.target, T, N * 4);
        rows(zb, a.behaviour, T, N * 4);
        rows(sact, a.action, T, 8);
        rows(sv, a.value, T + 1, 4);
        rows(sr, a.reward, T, 4);
        if (has_w) rows(sw, a.weight, T, 4);
        cpa_commit();
        cpa_wait<0>();
    }
    __syncthreads();
    // ---- phase A -----------------------------------------------------------------------------------------------------------
    for (int e = tid; e < E; e += VR_NT) {
        const int c = e % TC;
        if (c >= W) continue;
        const float* z = zt + (size_t)e * N;
        float* zo_ = zb + (size_t)e * N;
        const int act = (int)sact[e];
        float m = kF32Min, sum = 0.f, u2 = 0.f, mb = kF32Min, sb = 0.f;
        const float zta = z[act], zba = zo_[act];
        if (NC) {
            float zz[NR], zo[NR];
            load_row<NR>(z, zz);
            load_row<NR>(zo_, zo);
#pragma unroll
            for (int k = 0; k < NR; ++k) { m = fmaxf(m, zz[k]); mb = fmaxf(mb, zo[k]); }
            const float m2 = m * kLog2e, mb2 = mb * kLog2e;
#pragma unroll
            for (int k = 0; k < NR; ++k) {
                const float t = fmaxf(fmaf(zz[k], kLog2e, -m2), kF32Min);
                const float ex = ex2f_(t);
                sum += ex;
                u2 = fmaf(ex, t, u2);
                sb += ex2f_(fmaf(zo[k], kLog2e, -mb2));
            }
        } else {
            for (int k = 0; k < N; ++k) { m = fmaxf(m, z[k]); mb = fmaxf(mb, zo_[k]); }
            const float m2 = m * kLog2e, mb2 = mb * kLog2e;
            for (int k = 0; k < N; ++k) {
                const float t = fmaxf(fmaf(z[k], kLog2e, -m2), kF32Min);
                const float ex = ex2f_(t);
                sum += ex;
                u2 = fmaf(ex, t, u2);
                sb += ex2f_(fmaf(zo_[k], kLog2e, -mb2));
            }
        }
        const float l2s = lg2f_(sum);
        const float lse = m + l2s * kLn2;
        const float ent = (l2s - u2 * rcpf_(sum)) * kLn2;
        const float lp = zta - lse;
        const float lp_b = (zba - mb) - lg2f_(sb) * kLn2;
        sis[e] = ex2f_((lp - lp_b) * kLog2e);
        zo_[0] = lse;  // the behaviour row is dead: park the two statistics phase B needs (N >= 2)
        zo_[1] = ent;
    }
    __syncthreads();
    // ---- scan (vtrace.py:22-29): lane = column ------------------------------------------------------------------------------
    if (tid < W) {
        const int c = tid;
        float carry = 0.f, above = sv[T * TC + c];
        svs[T * TC + c] = above;  // vs_T = V_T
        if (GRADS) a.grad_value[(long long)T * B + c0 + c] = 0.f;
        int t1 = T;
        for (; t1 >= 16; t1 -= 16) {
            const int t0 = t1 - 16;
            float d[16], g[16], vv[17];
#pragma unroll
            for (int k = 0; k <= 16; ++k) vv[k] = sv[(t0 + k) * TC + c];
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float is = sis[(t0 + k) * TC + c], rw = sr[(t0 + k) * TC + c];
                d[k] = fmul(fminf(is, a.rho_clip), fsub(fadd(rw, fmul(a.gamma, vv[k + 1])), vv[k]));
                g[k] = fmul(a.gamma_lambda, fminf(is, a.c_clip));
            }
#pragma unroll
            for (int k = 15; k >= 0; --k) {
                carry = fadd(d[k], fmul(g[k], carry));
                vv[k] = fadd(vv[k], carry);
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) svs[(t0 + k) * TC + c] = vv[k];
        }
        for (int t = t1 - 1; t >= 0; --t) {
            const int e = t * TC + c;
            const float is = sis[e], v = sv[e];
            const float dl = fmul(fminf(is, a.rho_clip), fsub(fadd(sr[e], fmul(a.gamma, sv[e + TC])), v));
            carry = fadd(dl, fmul(fmul(a.gamma_lambda, fminf(is, a.c_clip)), carry));
            svs[e] = fadd(v, carry);
        }
    }
    __syncthreads();
    // ---- phase B -----------------------------------------------------------------------------------------------------------
    float acc[3] = {0.f, 0.f, 0.f};
    const float inv_m = 1.f / (float)((long long)T * B);
    for (int e = tid; e < E; e += VR_NT) {
        const int t = e / TC, c = e - t * TC;
        if (c >= W) continue;
        const float* z = zt + (size_t)e * N;
        const float lse = zb[(size_t)e * N], ent = zb[(size_t)e * N + 1];
        const int act = (int)sact[e];
        const float lp = z[act] - lse;
        const float is = sis[e];
        const float v = sv[e], rw = sr[e];
        const float w = has_w ? sw[e] : 1.f;
        const float adv = fmul(fminf(is, a.rho_pg_clip), fsub(fadd(rw, fmul(a.gamma, svs[e + TC])), v));
        const float dv = v - svs[e];
        acc[0] += lp * adv * w;
        acc[1] += dv * dv * w;
        acc[2] += ent * w;
        if (GRADS) {
            const long long g = (long long)t * B + c0 + c;
            const float c_act = g_pg * (-adv * w) * inv_m, c_ent = g_ent * w * inv_m;
            float* gz = a.grad_logit + g * N;
            if (NC) {
                float zz[NR], gj[NR];
                load_row<NR>(z, zz);
#pragma unroll
                for (int k = 0; k < NR; ++k) {
                    const float lpk = fmaxf(zz[k] - lse, kF32Min);
                    const float p = ex2f_(lpk * kLog2e);
                    gj[k] = -c_act * p - c_ent * p * (lpk + ent);
                    if (k == act) gj[k] += c_act;
                }
                store_row<NR>(gz, gj);
            } else {
                for (int k = 0; k < N; ++k) {
                    const float lpk = fmaxf(z[k] - lse, kF32Min);
                    const float p = ex2f_(lpk * kLog2e);
                    float gk = -c_act * p - c_ent * p * (lpk + ent);
                    if (k == act) gk += c_act;
                    gz[k] = gk;
                }
            }
            a.grad_value[g] = g_val * (2.f * w * dv * inv_m);
        }
    }
    if (!a.rec.verify) grid_store_partials<3, VR_NT>(acc, ws);  // summed by finalize_sums_kernel
}

static int g_vt_impl = 0;  // b200rl_vtrace_set_impl: 0 = automatic, 1 = streaming column tiles only, 2 = resident tiles first
// widest tile that leaves at least two CTAs per SM (227 KB of shared memory per SM, 1 KB reserved per CTA); 0 = no fit
static int vr_pick_tc(const VtFusedArgs& a) {
    if (g_vt_impl == 1 || a.N < 2) return 0;
    const bool has_w = a.weight != nullptr;
    if (a.B % 8 == 0 && vr_smem_bytes(a.T, a.N, has_w, 8) <= 112 * 1024) return 8;
    if (vr_smem_bytes(a.T, a.N, has_w, 4) <= 112 * 1024) return 4;
    return 0;
}

template <int NC, bool GRADS, int TC>
static int launch_vtres(const VtFusedArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    const size_t smem = vr_smem_bytes(a.T, a.N, a.weight != nullptr, TC);
    constexpr auto kern = vtrace_res_kernel<NC, GRADS, TC>;
    if (int rc = smem_opt_in<kern>(smem)) return rc;
    const long long grid = (a.B + TC - 1) / TC;
    if (ws_bytes < WS_MIN_BYTES || !ws_partials_fit((long long)(grid * 3), ws_bytes)) return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, VR_NT, smem, st, a, ws)) return rc;
    if (a.rec.verify) return B200RL_OK;
    return launch_finalize(ws, out, vtrace_finalize_args(a.T, a.B, (int)grid), st);
}

template <bool GRADS, int TC>
static int dispatch_vtres(const VtFusedArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    return with_nc(a.N, [&](auto nc) { return launch_vtres<nc, GRADS, TC>(a, out, ws, ws_bytes, st); });
}


static bool vt_layout_ok(const VtFusedArgs& a) {
    const bool al = aligned16(a.target) && aligned16(a.behaviour) && aligned16(a.action) && aligned16(a.value) &&
                    aligned16(a.reward) && (!a.weight || aligned16(a.weight)) &&
                    (!a.grad_logit || (aligned16(a.grad_logit) && aligned16(a.grad_value)));
    return al && a.N >= 1 && a.T >= 1 && a.B >= 4 && (a.B % 4) == 0;
}
// streaming column tiles (any T): the stage ring has to fit twice per SM
static bool vtws_ok(const VtFusedArgs& a) {
    return vt_layout_ok(a) && a.N <= 32 && vw_pick_stages(a.N, a.weight != nullptr) >= 3;
}
// resident tiles (short T): tile width, 0 = does not fit
static int vtres_tc(const VtFusedArgs& a) {
    if (!vt_layout_ok(a) || a.T > (1 << 20)) return 0;
    const int tc = vr_pick_tc(a);
    if (tc && WS_CTRL_WORDS + (a.B + tc - 1) / tc * 3 > WS_PARTIAL_LIMIT_WORDS) return 0;
    return tc;
}

template <int NC, bool GRADS, int TC>
static int launch_vtws(const VtFusedArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    const int stages = vw_pick_stages(a.N, a.weight != nullptr, TC);
    const size_t smem = vw_smem(a.N, a.weight != nullptr, stages, TC);
    constexpr auto kern = vtrace_ws_kernel<NC, GRADS, TC>;
    int sm_count, per_sm;
    if (int rc = resident_ctas<kern>(VW_THREADS, smem, sm_count, per_sm)) return rc;
    const long long n_tiles = (a.B + TC - 1) / TC;
    long long grid = (long long)sm_count * per_sm;
    if (grid > n_tiles) grid = n_tiles;
    if (ws_bytes < WS_MIN_BYTES || !ws_partials_fit((long long)(grid * 3), ws_bytes))
        return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, VW_THREADS, smem, st, a, ws, stages)) return rc;
    if (a.rec.verify) return B200RL_OK;
    return launch_finalize(ws, out, vtrace_finalize_args(a.T, a.B, (int)grid), st);
}

template <bool GRADS>
static int dispatch_vtws(const VtFusedArgs& a, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    // 32-column tiles when the 16-column tiles would not all be resident at once (two CTAs per SM)
    const bool wide = (a.B + 15) / 16 > 2 * NUM_SMS && a.B >= 32;
    return with_nc(a.N, [&](auto nc) {
        if (wide) return launch_vtws<nc, GRADS, 32>(a, out, ws, ws_bytes, st);
        return launch_vtws<nc, GRADS, 16>(a, out, ws, ws_bytes, st);
    });
}

}  // namespace b200rl

using namespace b200rl;

static void fill_vt(VtFusedArgs& a, const float* target_output, const float* behaviour_output, const long long* action,
                    const float* value, const float* reward, const float* weight, long long T, long long B, long long N,
                    double gamma, double lambda_, double rho, double c, double rho_pg) {
    a.target = target_output; a.behaviour = behaviour_output; a.action = action; a.value = value; a.reward = reward;
    a.weight = weight; a.T = T; a.B = B; a.N = (int)N; a.gamma = (float)gamma;
    a.gamma_lambda = (float)(gamma * lambda_);  // `factor = gamma * lambda_` in python double, vtrace.py:23
    a.rho_clip = (float)rho; a.c_clip = (float)c; a.rho_pg_clip = (float)rho_pg;
    a.trace = trace_enabled();
}

extern "C" int b200rl_vtrace_set_impl(int impl) {
    if (impl < 0 || impl > 2) return B200RL_ERR_ARG;
    const int old = g_vt_impl;
    g_vt_impl = impl;
    return old;
}

extern "C" int b200rl_vtrace_fused_supported(const float* target_output, const float* behaviour_output,
                                             const long long* action, const float* value, const float* reward,
                                             const float* weight, long long T, long long B, long long N,
                                             const float* grad_target_output, const float* grad_value) {
    if (!target_output || !behaviour_output || !action || !value || !reward || T < 1 || B < 1 || N < 1) return 0;
    VtFusedArgs a{};
    fill_vt(a, target_output, behaviour_output, action, value, reward, weight, T, B, N, 0.99, 0.95, 1.0, 1.0, 1.0);
    a.grad_logit = const_cast<float*>(grad_target_output);
    a.grad_value = const_cast<float*>(grad_value);
    return (vtres_tc(a) || vtws_ok(a)) ? 1 : 0;
}

extern "C" int b200rl_vtrace_fwd_grad(const float* target_output, const float* behaviour_output, const long long* action,
                                      const float* value, const float* reward, const float* weight, long long T,
                                      long long B, long long N, double gamma, double lambda_, double rho_clip_ratio,
                                      double c_clip_ratio, double rho_pg_clip_ratio, const float* g_expected,
                                      int verify, const float* g_policy, const float* g_value, const float* g_entropy,
                                      float* g_used, float* g_hint, float* out3, float* grad_target_output,
                                      float* grad_value, float* workspace, size_t workspace_bytes, void* stream) {
    if (!target_output || !behaviour_output || !action || !value || !reward || !workspace || T < 1 || B < 1 || N < 1)
        return B200RL_ERR_ARG;
    const bool grads = grad_target_output != nullptr;
    if (!upstream_args_ok(verify, out3, grads, grads && grad_value, g_expected, g_used)) return B200RL_ERR_ARG;
    VtFusedArgs a{};
    fill_vt(a, target_output, behaviour_output, action, value, reward, weight, T, B, N, gamma, lambda_, rho_clip_ratio,
            c_clip_ratio, rho_pg_clip_ratio);
    a.rec = verify ? verify_record(g_policy, g_value, g_entropy, nullptr, g_used, g_hint)
                   : forward_record(g_expected, g_used);
    a.grad_logit = grad_target_output; a.grad_value = grad_value;
    cudaStream_t st = (cudaStream_t)stream;
    // streaming column tiles wherever they fit (faster: they overlap loads with the scan); resident tiles take the shapes
    // they cannot (N > 15: no three-stage ring), and every shape they fit under b200rl_vtrace_set_impl(2)
    const int rtc = (vtws_ok(a) && g_vt_impl != 2) ? 0 : vtres_tc(a);
    if (rtc == 8)
        return grads ? dispatch_vtres<true, 8>(a, out3, workspace, workspace_bytes, st)
                     : dispatch_vtres<false, 8>(a, out3, workspace, workspace_bytes, st);
    if (rtc == 4)
        return grads ? dispatch_vtres<true, 4>(a, out3, workspace, workspace_bytes, st)
                     : dispatch_vtres<false, 4>(a, out3, workspace, workspace_bytes, st);
    if (!vtws_ok(a)) return B200RL_ERR_ARG;
    return grads ? dispatch_vtws<true>(a, out3, workspace, workspace_bytes, st)
                 : dispatch_vtws<false>(a, out3, workspace, workspace_bytes, st);
}
