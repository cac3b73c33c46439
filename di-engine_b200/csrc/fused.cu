// One-pass learner step: GAE scan + ppo_error forward (+ gradients) in ONE launch -- the metric of record
// "GAE + ppo_error on a (T, B) batch" without the two extra launches, their ramp-up/tail, and the separate latency chain
// of the scan.  Results are those of b200rl_gae followed by b200rl_ppo_fwd_grad (bit-identical adv, same loss/grad code).
//
// A persistent grid of 160-thread CTAs runs two phases:
//   G  CTAs with blockIdx < B/16 each run the warp-specialised GAE column-tile scan of gae_tile.cuh (4 loader warps,
//      1 scan warp).  The scan walks T from the newest row down, so the advantage rows appear newest-first; after every
//      32-row chunk the scan warp publishes "chunk k of this column tile is in HBM/L2" with a fence + one atomic on a
//      per-chunk counter.
//   P  every CTA (the others immediately, the GAE CTAs when their tile is done) runs the TMA-pipelined PPO tile loop of
//      ppo.cu, with two changes: tiles are handed out by an atomic counter in DESCENDING row order (newest time steps
//      first, matching the order in which advantages become available), and the per-row advantage is not part of the
//      TMA stage until the producer lane has seen the chunk counter of the tile's oldest time step reach the number of
//      column tiles (after the scan has finished this never waits again: the loop is then exactly ppo.cu's pipeline).
// No deadlock: phase G never waits for anything, its CTAs have the lowest block indices (scheduled first), and the grid
// never exceeds what the device can hold resident.
#include "../../include/b200rl.h"
#include "gae_tile.cuh"
#include "ppo_math.cuh"
#include "fused_args.cuh"

namespace b200rl {

constexpr int FUSED_TC = 16;                                  // GAE columns per tile: (16/4 + 1) warps == PPO_THREADS
constexpr int WS_TILE_CTR = 1;                                // control word: next PPO tile
constexpr int WS_CHUNK_CTR_WORDS = 4096;                      // per-chunk completion counters (T <= 131072)
constexpr int WS_CHUNK_CTR_OFF = (int)(WS_MIN_BYTES / 4) - WS_CHUNK_CTR_WORDS;
static_assert((FUSED_TC / 4 + 1) * 32 == PPO_THREADS, "GAE tile roles must fill the PPO CTA exactly");

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

template <int NC, bool GRADS, int RPT>
__global__ void __launch_bounds__(PPO_THREADS, 4) gae_ppo_kernel(FusedArgs f, float* out, float* ws) {
    pdl_prologue();
    constexpr int PPO_R = PPO_CT * RPT;  // rows per PPO tile
    extern __shared__ __align__(128) unsigned char smem[];
    const PpoArgs& a = f.p;
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x;
    const int wid = tid >> 5, lane = tid & 31;
    const bool is_producer = wid == PPO_CW;
    const bool has_pre = a.logit_pre != nullptr, has_w = a.weight != nullptr;
    const PpoTileLayout L = ppo_layout(N, has_pre, has_w, PPO_R);
    const int warp_out_bytes = 32 * RPT * N * 4;
    unsigned char* outbuf = smem + PPO_STAGES * L.stage_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + (GRADS ? PPO_OUTBUFS * L.logit_bytes : 0));
    uint64_t* empty = full + PPO_STAGES;
    int* tile_slot = reinterpret_cast<int*>(empty + PPO_STAGES);
    unsigned int* ctrl = reinterpret_cast<unsigned int*>(ws);
    unsigned int* chunk_ctr = ctrl + WS_CHUNK_CTR_OFF;

    float g[4] = {0.f, 0.f, 0.f, 0.f};
    if (GRADS) upstream<4>(a.rec, false, ppo_owned(a), g);  // a forward launch: records `used`, never skips
    const PpoUpstream up{g[0], g[1], g[2], g[3], 1.f / (float)a.S};

    // ---- phase G: GAE column tiles (shared memory aliased onto the not-yet-used PPO stage ring) -----------------------
    const long long n_col_tiles = (f.B + FUSED_TC - 1) / FUSED_TC;
    // completion counters: one per (32-row chunk, group of PPO_R columns) when the PPO tiles line up with the columns
    // (B % PPO_R == 0: a tile = one time step x one column group, so it only waits for ITS columns), else one per chunk
    const bool fine = (f.B % PPO_R) == 0;
    const long long n_groups = fine ? f.B / PPO_R : 1;
    const unsigned int group_need = fine ? (unsigned int)(PPO_R / FUSED_TC) : (unsigned int)n_col_tiles;
    {
        auto s_d = reinterpret_cast<float (*)[GAE_CH][FUSED_TC]>(smem);
        auto s_f = s_d + GAE_NCHUNK;
        for (long long ct = blockIdx.x; ct < n_col_tiles; ct += gridDim.x) {
            gae_tile_body<FUSED_TC, true>(f.value, f.next_value, f.reward, f.done, f.traj, a.adv_out, f.T, f.B, 1,
                                          f.gamma, f.gl, f.mask_inplace, ct * FUSED_TC, s_d, s_f,
                                          [&](long long gk, bool any) {
                                              if (!any) return;
                                              fence_acq_rel_gpu();  // this lane's adv stores are visible device-wide ...
                                              __syncwarp();
                                              if (lane == 0) {
                                                  const long long grp = fine ? (ct * FUSED_TC) / PPO_R : 0;
                                                  atomicAdd(&chunk_ctr[gk * n_groups + grp], 1u);  // ... before the count
                                              }
                                          });
            __syncthreads();
        }
    }

    // ---- phase P: PPO tiles, newest rows first ------------------------------------------------------------------------
    const long long n_full = a.S / PPO_R;
    const int tail_rows = (int)(a.S - n_full * PPO_R);
    const long long n_tiles = n_full + (tail_rows ? 1 : 0);
    if (tid == 0) {
        for (int s = 0; s < PPO_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], PPO_CW);
        }
        mbar_fence_init();
    }
    __syncthreads();

    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (is_producer) {
        if (lane == 0) {
            long long ready_upto = -1;  // GAE chunks [0, ready_upto] are known complete for every column tile
            long long tix = (long long)atomicAdd(&ctrl[WS_TILE_CTR], 1u);
            for (int i = 0;; ++i) {
                const int sg = i % PPO_STAGES;
                if (i >= PPO_STAGES) mbar_wait(&empty[sg], (uint32_t)(((i / PPO_STAGES) - 1) & 1));
                if (tix >= n_tiles) {
                    tile_slot[sg] = -1;
                    mbar_arrive(&full[sg]);
                    break;
                }
                const long long t = n_tiles - 1 - tix;
                const long long row0 = t * PPO_R;
                // the oldest time step of this tile decides which GAE chunk must be complete before adv is read;
                // tiles come newest-first, so after the scan has finished this never waits again
                const long long need = (f.T - 1 - row0 / f.B) / GAE_CH;
                tile_slot[sg] = (int)t;
                const bool full_tile = t < n_full;
                unsigned char* st = smem + sg * L.stage_bytes;
                uint64_t* bar = &full[sg];
                if (full_tile) {  // everything that does not depend on the scan starts streaming right away
                    mbar_expect_tx(bar, (uint32_t)L.tx_bytes);
                    tma_load_1d(st, a.logit_new + row0 * N, L.logit_bytes, bar);
                    tma_load_1d(st + L.off_old, a.logit_old + row0 * N, L.logit_bytes, bar);
                    if (has_pre) tma_load_1d(st + L.off_pre, a.logit_pre + row0 * N, L.logit_bytes, bar);
                    tma_load_1d(st + L.off_act, a.action + row0, PPO_R * 8, bar);
                    tma_load_1d(st + L.off_vn, a.value_new + row0, PPO_R * 4, bar);
                    tma_load_1d(st + L.off_vo, a.value_old + row0, PPO_R * 4, bar);
                    tma_load_1d(st + L.off_ret, a.ret + row0, PPO_R * 4, bar);
                    if (has_w) tma_load_1d(st + L.off_w, a.weight + row0, PPO_R * 4, bar);
                }
                if (need > ready_upto) {
                    const long long grp = fine ? (row0 % f.B) / PPO_R : 0;
                    while (ld_acquire_u32(&chunk_ctr[need * n_groups + grp]) < group_need) __nanosleep(32);
                    if (!fine) ready_upto = need;  // per-chunk counters are monotone in tile order; per-group ones are not
                    asm volatile("fence.proxy.async;" ::: "memory");  // order the TMA reads of adv after the acquire
                }
                if (full_tile) tma_load_1d(st + L.off_adv, a.adv + row0, PPO_R * 4, bar);  // completes the stage
                else mbar_arrive(bar);  // ragged newest tile: its consumers use plain loads
                tix = (long long)atomicAdd(&ctrl[WS_TILE_CTR], 1u);  // next tile: the round trip overlaps the stage wait
            }
        }
    } else {
        for (int i = 0;; ++i) {
            const int sg = i % PPO_STAGES;
            unsigned char* st = smem + sg * L.stage_bytes;
            mbar_wait(&full[sg], (uint32_t)((i / PPO_STAGES) & 1));
            const long long t = tile_slot[sg];
            if (t < 0) break;
            const long long row0 = t * PPO_R;
            const bool full_tile = t < n_full;
            float* gtile = reinterpret_cast<float*>(outbuf + (wid * 2 + (i & 1)) * warp_out_bytes) - wid * 32 * RPT * N;
#pragma unroll
            for (int q = 0; q < RPT; ++q) {
                const int rit = (wid * RPT + q) * 32 + lane;  // row in tile: a warp covers 32*RPT consecutive rows
                float adv = 0.f;
                if (full_tile) {
                    adv = reinterpret_cast<const float*>(st + L.off_adv)[rit];
                } else if (rit < tail_rows) {
                    // ragged newest tile: plain loads into this thread's own slots; the producer saw its chunk complete
                    adv = __ldcg(a.adv + row0 + rit);
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
                    reinterpret_cast<float*>(st + L.off_ret)[rit] = a.ret[row0 + rit];
                    if (has_w) reinterpret_cast<float*>(st + L.off_w)[rit] = a.weight[row0 + rit];
                }
                if (full_tile || rit < tail_rows)
                    ppo_row_compute<NC, true, GRADS>(a, L, st, rit, N, adv, full_tile, gtile, row0, up, acc);
            }
            if (GRADS && full_tile) {
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                    tma_store_1d(a.grad_logit + (row0 + wid * 32 * RPT) * N, gtile + wid * 32 * RPT * N,
                                 warp_out_bytes);
                    tma_store_commit();
                    tma_store_wait_read<1>();
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[sg]);
        }
        if (GRADS && lane == 0) tma_store_wait_read<0>();
    }

    grid_store_partials<6, PPO_THREADS>(acc, ws);  // summed (and the scheduling counters cleared) by finalize_sums_kernel
}

static bool fused_ok(const FusedArgs& f) {
    const PpoArgs& a = f.p;
    const bool al = aligned16(a.logit_new) && aligned16(a.logit_old) && (!a.logit_pre || aligned16(a.logit_pre)) &&
                    aligned16(a.action) && aligned16(a.value_new) && aligned16(a.value_old) && aligned16(a.ret) &&
                    (!a.weight || aligned16(a.weight)) && (!a.grad_logit || aligned16(a.grad_logit)) &&
                    aligned16(f.value) && aligned16(f.next_value) && aligned16(f.reward) && aligned16(a.adv) &&
                    (!f.done || aligned16(f.done)) && (!f.traj || aligned16(f.traj));
    return al && a.N >= 1 && a.N <= 32 && f.T >= 1 && f.B >= 4 && (f.B % 4) == 0 && f.T * f.B == a.S &&
           ((f.T + GAE_CH - 1) / GAE_CH) * ((f.B + PPO_CT - 1) / PPO_CT) <= WS_CHUNK_CTR_WORDS;
}

// dynamic shared memory of gae_ppo_kernel: PPO stage ring, gradient tiles, barriers and tile slots
static size_t fused_smem(const FusedArgs& f, bool grads, int rpt) {
    const PpoTileLayout L = ppo_layout(f.p.N, f.p.logit_pre != nullptr, f.p.weight != nullptr, PPO_CT * rpt);
    size_t smem = (size_t)PPO_STAGES * L.stage_bytes + (grads ? (size_t)PPO_OUTBUFS * L.logit_bytes : 0) +
                  2 * PPO_STAGES * sizeof(uint64_t) + PPO_STAGES * sizeof(int) + 16;
    const size_t gae_smem = (size_t)2 * GAE_NCHUNK * GAE_CH * FUSED_TC * sizeof(float);
    if ((size_t)PPO_STAGES * L.stage_bytes < gae_smem) smem += gae_smem;  // keep the aliased GAE arrays inside the ring
    return smem;
}

template <int NC, bool GRADS, int RPT>
static int launch_fused(const FusedArgs& f, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    constexpr int PPO_R = PPO_CT * RPT;
    const PpoArgs& a = f.p;
    const size_t smem = fused_smem(f, GRADS, RPT);
    constexpr auto kern = gae_ppo_kernel<NC, GRADS, RPT>;
    if (smem > 227 * 1024) return B200RL_ERR_ARG;
    int sm_count, per_sm;
    if (int rc = resident_ctas<kern>(PPO_THREADS, smem, sm_count, per_sm)) return rc;
    const long long n_tiles = (a.S + PPO_R - 1) / PPO_R;
    long long grid = (long long)sm_count * per_sm;  // never more than can be resident (phase P spins on phase G)
    if (grid > n_tiles) grid = n_tiles;
    if (grid < 1) grid = 1;
    if (!ws_partials_fit((long long)(grid * 6), ws_bytes)) return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, PPO_THREADS, smem, st, f, out, ws)) return rc;
    FinalizeArgs fa = ppo_finalize_args(a.S, a.logit_pre != nullptr, (int)grid);
    fa.clear_ctrl_from = WS_TILE_CTR; fa.clear_ctrl_n = 1;
    const long long n_groups = (f.B % PPO_R) == 0 ? f.B / PPO_R : 1;
    fa.clear_tail_off = WS_CHUNK_CTR_OFF;
    fa.clear_tail_n = (int)(((f.T + GAE_CH - 1) / GAE_CH) * n_groups);
    return launch_finalize(ws, out, fa, st);
}

template <bool GRADS>
static int dispatch_fused(const FusedArgs& f, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    // 2 rows per thread once there are four 256-row tiles per SM, where their layout fits; 1 row fits for every N <= 32.
    // The TMA issue rate per SM is bounded per operation, so 256-row tiles double the bytes each bulk copy moves.
    const int rpt = (f.p.S >= 256LL * NUM_SMS * 4 && fused_smem(f, GRADS, 2) <= 227 * 1024) ? 2 : 1;
    return with_nc(f.p.N, [&](auto nc) {
        if (rpt == 2) return launch_fused<nc, GRADS, 2>(f, out, ws, ws_bytes, st);
        return launch_fused<nc, GRADS, 1>(f, out, ws, ws_bytes, st);
    });
}

}  // namespace b200rl

using namespace b200rl;

static void fill_fused(FusedArgs& f, const float* value, float* next_value, const float* reward, const float* done,
                       const float* traj_flag, long long T, long long B, double gamma, double lambda_,
                       int mask_inplace, const float* logit_new, const float* logit_old,
                       const float* logit_pretrained, const long long* action, const float* value_new,
                       const float* value_old, const float* return_, const float* weight, long long N,
                       double clip_ratio, int use_value_clip, double dual_clip, int kl_type, float* adv) {
    PpoArgs& a = f.p;
    a.logit_new = logit_new; a.logit_old = logit_old; a.logit_pre = logit_pretrained; a.action = action;
    a.value_new = value_new; a.value_old = value_old; a.adv = adv; a.adv_out = adv; a.ret = return_; a.weight = weight;
    a.S = T * B; a.G = 1; a.N = (int)N; a.clip = (float)clip_ratio; a.clip_lo = (float)(1.0 - clip_ratio);
    a.clip_hi = (float)(1.0 + clip_ratio); a.dual_clip = (float)dual_clip; a.use_value_clip = use_value_clip;
    a.kl_type = kl_type;
    f.value = value; f.next_value = next_value; f.reward = reward; f.done = done; f.traj = traj_flag; f.T = T; f.B = B;
    f.gamma = (float)gamma; f.gl = (float)(gamma * lambda_); f.mask_inplace = mask_inplace;
    f.trace = trace_enabled();
}

extern "C" int b200rl_gae_ppo_supported(const float* value, const float* next_value, const float* reward,
                                        const float* done, const float* traj_flag, long long T, long long B,
                                        const float* logit_new, const float* logit_old,
                                        const float* logit_pretrained, const long long* action,
                                        const float* value_new, const float* value_old, const float* return_,
                                        const float* weight, long long N, const float* adv,
                                        const float* grad_logit_new) {
    FusedArgs f{};
    fill_fused(f, value, const_cast<float*>(next_value), reward, done, traj_flag, T, B, 0.99, 0.95, 0, logit_new,
               logit_old, logit_pretrained, action, value_new, value_old, return_, weight, N, 0.2, 1, 0.0, 1,
               const_cast<float*>(adv));
    f.p.grad_logit = const_cast<float*>(grad_logit_new);
    if (!value || !next_value || !reward || !logit_new || !logit_old || !action || !value_new || !value_old ||
        !return_ || !adv)
        return 0;
    return (fused_ok(f) || colws_ok(f)) ? 1 : 0;
}

// kernel of the one-launch step: 0 = automatic, 1 = row tiles with chunk counters (gae_ppo_kernel, this file),
// 2 = column tiles (colws.cu).  Either falls back to the other where it cannot take the call.
static int g_impl = 0;
extern "C" int b200rl_gae_ppo_set_impl(int impl) {
    if (impl < 0 || impl > 2) return B200RL_ERR_ARG;
    const int old = g_impl;
    g_impl = impl;
    return old;
}

static int gae_ppo_step(const float* value, float* next_value, const float* reward, const float* done,
                        const float* traj_flag, long long T, long long B, double gamma, double lambda_,
                        int mask_next_value_inplace, const float* logit_new, const float* logit_old,
                        const float* logit_pretrained, const long long* action, const float* value_new,
                        const float* value_old, const float* return_, const float* weight, long long N,
                        double clip_ratio, int use_value_clip, double dual_clip, int kl_type, const float* g_expected,
                        float* g_used, float* adv, float* out, float* grad_logit_new, float* grad_value_new,
                        const unsigned long long* mailbox_ptrs_dev, int rank, int world, unsigned int* seq_dev,
                        float* out_mean, float* workspace, size_t workspace_bytes, void* stream) {
    const bool grads = g_expected != nullptr;
    if (!value || !next_value || !reward || !logit_new || !logit_old || !action || !value_new || !value_old ||
        !return_ || !adv || !workspace || T < 1 || B < 1 || N < 1 || kl_type < 1 || kl_type > 3 ||
        !upstream_args_ok(0, out, grads, grad_logit_new && grad_value_new, g_expected, g_used))
        return B200RL_ERR_ARG;
    FusedArgs f{};
    fill_fused(f, value, next_value, reward, done, traj_flag, T, B, gamma, lambda_, mask_next_value_inplace,
               logit_new, logit_old, logit_pretrained, action, value_new, value_old, return_, weight, N, clip_ratio,
               use_value_clip, dual_clip, kl_type, adv);
    if (grads) {
        f.p.rec = forward_record(g_expected, g_used);
        f.p.grad_logit = grad_logit_new; f.p.grad_value = grad_value_new;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const bool row_ok = fused_ok(f), col_ok = colws_ok(f);
    if (!row_ok && !col_ok) return B200RL_ERR_ARG;
    if (mailbox_ptrs_dev) {  // data-parallel exchange in the epilogue of the column-tile kernel
        if (!seq_dev || !out_mean || world < 1 || world > 32 || rank < 0 || rank >= world || !col_ok)
            return B200RL_ERR_ARG;
        f.x_mailboxes = mailbox_ptrs_dev; f.x_seq = seq_dev; f.x_out_mean = out_mean; f.x_rank = rank; f.x_world = world;
        return launch_colws(f, grads, out, workspace, workspace_bytes, st);
    }
    // column tiles need enough columns to fill the machine (64 CTAs of 16 columns); tiny problems are launch-bound either
    // way.  colws.cu takes 32-column tiles only where they give nearly every SM one (B >= 3940 on an H100's 132 SMs), far
    // above this threshold, so it is derived for its 16-column geometry
    const bool want_col = g_impl == 2 || (g_impl == 0 && (B >= 16 * 64 || T * B <= 16384));
    if (col_ok && (want_col || !row_ok)) return launch_colws(f, grads, out, workspace, workspace_bytes, st);
    return grads ? dispatch_fused<true>(f, out, workspace, workspace_bytes, st)
                 : dispatch_fused<false>(f, out, workspace, workspace_bytes, st);
}

extern "C" int b200rl_gae_ppo_fwd_grad(const float* value, float* next_value, const float* reward, const float* done,
                                       const float* traj_flag, long long T, long long B, double gamma,
                                       double lambda_, int mask_next_value_inplace, const float* logit_new,
                                       const float* logit_old, const float* logit_pretrained,
                                       const long long* action, const float* value_new, const float* value_old,
                                       const float* return_, const float* weight, long long N, double clip_ratio,
                                       int use_value_clip, double dual_clip, int kl_type, const float* g_expected,
                                       float* g_used, float* adv, float* out, float* grad_logit_new,
                                       float* grad_value_new, float* workspace, size_t workspace_bytes,
                                       void* stream) {
    return gae_ppo_step(value, next_value, reward, done, traj_flag, T, B, gamma, lambda_, mask_next_value_inplace,
                        logit_new, logit_old, logit_pretrained, action, value_new, value_old, return_, weight, N,
                        clip_ratio, use_value_clip, dual_clip, kl_type, g_expected, g_used, adv, out, grad_logit_new,
                        grad_value_new, nullptr, 0, 1, nullptr, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int b200rl_gae_ppo_fwd_grad_dp(const float* value, float* next_value, const float* reward, const float* done,
                                          const float* traj_flag, long long T, long long B, double gamma,
                                          double lambda_, int mask_next_value_inplace, const float* logit_new,
                                          const float* logit_old, const float* logit_pretrained,
                                          const long long* action, const float* value_new, const float* value_old,
                                          const float* return_, const float* weight, long long N, double clip_ratio,
                                          int use_value_clip, double dual_clip, int kl_type, const float* g_expected,
                                          float* g_used, float* adv, float* out, float* grad_logit_new,
                                          float* grad_value_new, const unsigned long long* mailbox_ptrs_dev, int rank,
                                          int world, unsigned int* seq_dev, float* out_mean, float* workspace,
                                          size_t workspace_bytes, void* stream) {
    if (!mailbox_ptrs_dev) return B200RL_ERR_ARG;
    return gae_ppo_step(value, next_value, reward, done, traj_flag, T, B, gamma, lambda_, mask_next_value_inplace,
                        logit_new, logit_old, logit_pretrained, action, value_new, value_old, return_, weight, N,
                        clip_ratio, use_value_clip, dual_clip, kl_type, g_expected, g_used, adv, out, grad_logit_new,
                        grad_value_new, mailbox_ptrs_dev, rank, world, seq_dev, out_mean, workspace, workspace_bytes,
                        stream);
}
