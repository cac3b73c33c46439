// Column-tile learner step, warp-specialised: gae -> ppo_error (+ gradients) in ONE launch, no cross-CTA dependency, no
// CTA-wide barrier in the loop, every copy a plain 16-byte LDGSTS (cp.async) issued by a dedicated loader warp.
//
// Why a loader warp rather than every thread copying: with all threads copying and a __syncthreads per chunk, about half
// of the instructions go to copy addressing and the kernel is issue-bound.  Why per-lane LDGSTS rather than 2-D TMA boxes:
// the TMA unit's issue cost is per operation, and a column tile of the (T, B) tensors gives 64-byte box rows, 2 KB per
// operation (57 operations per tile), so the copies wait on the TMA unit instead.
//
// A CTA owns TC = 16 batch columns for ALL T (the recurrence of gae.py:65-69 runs along T only, ppo.py:77-140 is pointwise).
// Time is walked newest-first in chunks of R = 16 steps (256 transitions).  Warp roles (10 warps, two CTAs per SM):
//   warp 8     loader: cp.async of the chunk's PPO inputs (logit_new | logit_old | action | value_new | value_old |
//              return_ [| weight | logit_pre]) into an S-stage ring (S = 4 at N = 6); completion arrives on the stage's
//              mbarrier (cp.async.mbarrier.arrive.noinc); a stage is refilled as soon as the consumers release it.
//   warp 9     scanner: own two-deep cp.async ring of the five GAE inputs; per chunk delta / f in the reference's operation
//              order, the in-place next_value mask (gae.py:61), the sequential scan A = delta + f*A (lane = column, separate
//              round-to-nearest mul and add: bit-identical to the torch loop); publishes the chunk's advantages in an
//              S-slot shared-memory ring (mbarrier) and writes them to HBM (16-byte coalesced).
//   warps 0-7  consumers: thread = transition; wait for "chunk landed" and "advantages ready", run ppo_row_compute_to (the
//              row code of ppo.cu) and store the gradient row and the value gradient straight to HBM; arrive on "done".
// Rings run across tile boundaries (static tile -> CTA assignment: deterministic loss partial sums).
//
// Once the ring is primed the chunks stream at the rate HBM delivers them; what separates the kernel from the roofline is
// the time until the first chunk has landed and the tail (last chunk's math, store drain, partial sums, finalize_sums
// launch).  Loader variants that were slower: loop-invariant piece offsets in registers with one or two loader warps (the
// faster refill issues the ring of every CTA in one burst, which delays chunk 0 and costs DRAM efficiency), the same with a
// throttled prologue, no unrolling of the copy loop, 2 or 3 ring stages.
//
// Algorithmic traffic: 24 B (GAE) + 104 B (ppo_error forward + gradients, N = 6) = 128 B per transition, each byte once.
#include "../../include/b200rl.h"
#include "fused_args.cuh"

namespace b200rl {

constexpr int CW_CW = 8;                  // consumer warps
constexpr int CW_CT = CW_CW * 32;         // consumer threads = transitions per chunk
constexpr int CW_THREADS = CW_CT + 64;    // + loader warp + scanner warp
constexpr int CW_TC = 16;                 // columns per tile
constexpr int CW_R = CW_CT / CW_TC;       // time steps per chunk (16)
constexpr int CW_MAX_STAGES = 4;
constexpr int CW_RAW_ARR = CW_R * CW_TC * 4;  // bytes of one raw GAE array chunk
constexpr int CW_RAW_BYTES = 5 * CW_RAW_ARR;  // value | next_value | reward | done | traj_flag

#define CW_TRACE(slot)                                                                                   \
    do {                                                                                                 \
        if (f.trace) reinterpret_cast<unsigned long long*>(ws + 65536)[blockIdx.x * 32 + (slot)] = gtimer(); \
    } while (0)

struct CwItem {
    long long tile;
    long long q;  // chunk from the top of the trajectory: time steps [T - (q+1)R, T - qR)
};

__host__ __device__ inline int cw_stage_bytes(int N, bool has_pre, bool has_w) {
    return (CW_CT * ((has_pre ? 3 : 2) * N * 4 + 8 + 12 + (has_w ? 4 : 0)) + 127) & ~127;
}

template <int NC, bool GRADS>
__global__ void __launch_bounds__(CW_THREADS, 2) gae_ppo_ws_kernel(FusedArgs f, float* ws, int n_stages) {
    // PDL: the next kernel may start launching right away; the wait for the previous kernels' results comes after the
    // barrier set-up below (nothing before it touches global memory except the optional trace stamp)
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ __align__(128) unsigned char smem[];
    const PpoArgs& a = f.p;
    const int N = NC ? NC : a.N;
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const bool has_pre = a.logit_pre != nullptr, has_w = a.weight != nullptr;
    PpoTileLayout L;
    {
        L.logit_bytes = CW_CT * N * 4;
        int o = L.logit_bytes;
        L.off_old = o; o += L.logit_bytes;
        L.off_pre = o; if (has_pre) o += L.logit_bytes;
        L.off_act = o; o += CW_CT * 8;
        L.off_vn = o; o += CW_CT * 4;
        L.off_vo = o; o += CW_CT * 4;
        L.off_adv = 0;
        L.off_ret = o; o += CW_CT * 4;
        L.off_w = o; if (has_w) o += CW_CT * 4;
        L.stage_bytes = (o + 127) & ~127;
        L.tx_bytes = o;
    }
    const int S = n_stages;
    unsigned char* raw = smem + S * L.stage_bytes;                                            // [2][5][R][TC]
    auto advr = reinterpret_cast<float (*)[CW_R][CW_TC]>(raw + 2 * CW_RAW_BYTES);            // [S][R][TC]
    auto fbuf = reinterpret_cast<float (*)[CW_TC]>(reinterpret_cast<unsigned char*>(advr) + CW_MAX_STAGES * CW_RAW_ARR);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(fbuf) + CW_RAW_ARR);
    uint64_t* full = bars;                           // [S] PPO chunk landed (32 loader-lane arrivals)
    uint64_t* done = bars + CW_MAX_STAGES;           // [S] consumers finished the chunk (CW_CW arrivals)
    uint64_t* adv_ready = bars + 2 * CW_MAX_STAGES;  // [S] advantages of the chunk are in advr[s]

    const long long T = f.T, B = f.B;
    const long long n_tiles = (B + CW_TC - 1) / CW_TC;
    const long long n_chunks = (T + CW_R - 1) / CW_R;
    const bool has_done = f.done != nullptr, has_traj = f.traj != nullptr;

    if (tid == 0) {
        CW_TRACE(0);
        for (int s = 0; s < CW_MAX_STAGES; ++s) {
            mbar_init(&full[s], 32);
            mbar_init(&done[s], CW_CW);
            mbar_init(&adv_ready[s], 1);
        }
        mbar_fence_init();
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    __syncthreads();
    // data-parallel training: consumer warp k of the first CTA consumes the loss scalar k of two steps ago from its mailbox and
    // publishes the previous step's (staged by its finalize launch) to the peers -- while it would otherwise just wait for its
    // first chunk; the NVLink acknowledgements return while this kernel streams (common.cuh)
    if (f.x_mailboxes && blockIdx.x == 0 && wid < 6) {
        XchgArgs x{f.x_mailboxes, f.x_seq, f.x_out_mean, f.x_rank, f.x_world};
        p2p_pipeline_warp(x, wid);
    }

    auto item_valid = [&](const CwItem& it) { return it.tile < n_tiles; };
    auto item_next = [&](CwItem& it) {
        if (++it.q >= n_chunks) {
            it.q = 0;
            it.tile += gridDim.x;
        }
    };
    const CwItem first{(long long)blockIdx.x, 0};
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};

    if (wid == CW_CW) {
        // =============================================== loader ===========================================================
        // R segments (one per time step) of `esz` bytes per column: P = TC*esz/16 pieces per segment in shared memory
        auto rows_of = [&](unsigned char* dst, const void* src, long long t0, long long c0, int esz, int jmin, int W) {
            const int P = CW_TC * esz / 16, Pv = W * esz / 16;
            const unsigned char* g = reinterpret_cast<const unsigned char*>(src) + (t0 * B + c0) * esz;
            const long long rstride = B * esz;
            const int n = CW_R * P;
#pragma unroll 4
            for (int p = lane; p < n; p += 32) {
                const int row = p / P, o = p - row * P;
                if (row >= jmin && o < Pv) cpa16(dst + p * 16, g + row * rstride + o * 16);
            }
        };
        // The FIRST stage of a CTA uses lane-owns-a-piece-column copies (common.cuh warp_copy_rows, ~3 instructions per copy),
        // every later one the flat loop (~35 instructions per copy).  The kernel streams at the HBM rate in steady state, so a
        // faster loader buys nothing there -- issued in bursts the copies only deepen the queues in front of everybody's next
        // chunk -- but the first stage is pure latency: the flat loop's address arithmetic runs before the first byte is
        // requested.
        CwItem it = first;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            if (j >= S) mbar_wait(&done[s], (uint32_t)(ph ^ 1));
            if (lane == 0 && j < 6) CW_TRACE(20 + 2 * j);
            const long long c0 = it.tile * CW_TC;
            const long long t0 = T - (it.q + 1) * CW_R;
            const int jmin = t0 < 0 ? (int)-t0 : 0;
            const int W = (int)((B - c0) < CW_TC ? (B - c0) : CW_TC);
            unsigned char* st = smem + s * L.stage_bytes;
            if (jmin == 0 && W == CW_TC && j == 0) {
                // full chunk of a full tile: a row segment is TC * esz / 16 = esz pieces (4 N | 8 | 4).  Logits and actions
                // go in 8-piece groups (a lane group covers one full 128-byte line per row: the 4-piece grouping doubles the
                // number of L2 requests, which makes it slower than the flat loop); the float tensors have 64-byte rows.
                const uint32_t sb = smem_u32(st);
                const long long e0 = t0 * B + c0;
                const long long ls = B * N * 4;
                if (N & 1) {
                    warp_copy_rows<4, CW_R, NC>(sb, a.logit_new + e0 * N, ls, N, lane);
                    warp_copy_rows<4, CW_R, NC>(sb + L.off_old, a.logit_old + e0 * N, ls, N, lane);
                    if (has_pre) warp_copy_rows<4, CW_R, NC>(sb + L.off_pre, a.logit_pre + e0 * N, ls, N, lane);
                    warp_copy_rows<4, CW_R, 2>(sb + L.off_act, a.action + e0, B * 8, 2, lane);
                } else {
                    warp_copy_rows<8, CW_R, NC / 2>(sb, a.logit_new + e0 * N, ls, N / 2, lane);
                    warp_copy_rows<8, CW_R, NC / 2>(sb + L.off_old, a.logit_old + e0 * N, ls, N / 2, lane);
                    if (has_pre) warp_copy_rows<8, CW_R, NC / 2>(sb + L.off_pre, a.logit_pre + e0 * N, ls, N / 2, lane);
                    warp_copy_rows<8, CW_R, 1>(sb + L.off_act, a.action + e0, B * 8, 1, lane);
                }
                warp_copy_rows<4, CW_R, 1>(sb + L.off_vn, a.value_new + e0, B * 4, 1, lane);
                warp_copy_rows<4, CW_R, 1>(sb + L.off_vo, a.value_old + e0, B * 4, 1, lane);
                warp_copy_rows<4, CW_R, 1>(sb + L.off_ret, a.ret + e0, B * 4, 1, lane);
                if (has_w) warp_copy_rows<4, CW_R, 1>(sb + L.off_w, a.weight + e0, B * 4, 1, lane);
            } else {
                rows_of(st, a.logit_new, t0, c0, N * 4, jmin, W);
                rows_of(st + L.off_old, a.logit_old, t0, c0, N * 4, jmin, W);
                if (has_pre) rows_of(st + L.off_pre, a.logit_pre, t0, c0, N * 4, jmin, W);
                rows_of(st + L.off_act, a.action, t0, c0, 8, jmin, W);
                rows_of(st + L.off_vn, a.value_new, t0, c0, 4, jmin, W);
                rows_of(st + L.off_vo, a.value_old, t0, c0, 4, jmin, W);
                rows_of(st + L.off_ret, a.ret, t0, c0, 4, jmin, W);
                if (has_w) rows_of(st + L.off_w, a.weight, t0, c0, 4, jmin, W);
            }
            cpa_mbar_arrive(&full[s]);
            if (lane == 0 && j < 6) CW_TRACE(21 + 2 * j);
            if (++s == S) { s = 0; ph ^= 1; }
            item_next(it);
        }
    } else if (wid == CW_CW + 1) {
        // =============================================== scanner ==========================================================
        auto issue_raw = [&](const CwItem& it, int slot) {
            const long long c0 = it.tile * CW_TC;
            const long long t0 = T - (it.q + 1) * CW_R;
            const int W = (int)((B - c0) < CW_TC ? (B - c0) : CW_TC);
            unsigned char* dst = raw + slot * CW_RAW_BYTES;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int p = lane + 32 * k;  // R*4 = 64 pieces per array
                const int row = p >> 2, o = p & 3;
                if (t0 + row >= 0 && o * 4 < W) {
                    const long long off = (t0 + row) * B + c0 + o * 4;
                    cpa16(dst + p * 16, f.value + off);
                    cpa16(dst + CW_RAW_ARR + p * 16, f.next_value + off);
                    cpa16(dst + 2 * CW_RAW_ARR + p * 16, f.reward + off);
                    if (has_done) cpa16(dst + 3 * CW_RAW_ARR + p * 16, f.done + off);
                    if (has_traj) cpa16(dst + 4 * CW_RAW_ARR + p * 16, f.traj + off);
                }
            }
        };
        CwItem it = first, pf = first;
        for (int k = 0; k < 2; ++k) {
            if (item_valid(pf)) {
                issue_raw(pf, k);
                item_next(pf);
            }
            cpa_commit();
        }
        float carry = 0.f;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            const long long c0 = it.tile * CW_TC;
            const long long t0 = T - (it.q + 1) * CW_R;
            const int slot = j & 1;
            if (it.q == 0) carry = 0.f;
            cpa_wait<1>();
            __syncwarp();
            if (j >= S) mbar_wait(&done[s], (uint32_t)(ph ^ 1));  // the consumers are through the chunk that used advr[s]
            float (*ab)[CW_TC] = advr[s];
            const float* rv = reinterpret_cast<const float*>(raw + slot * CW_RAW_BYTES);
            const float* rn = rv + CW_R * CW_TC;
            const float* rr = rn + CW_R * CW_TC;
            const float* rd = rr + CW_R * CW_TC;
            const float* rt = rd + CW_R * CW_TC;
            const int cq = (lane & 3) * 4;
#pragma unroll
            for (int p = 0; p < CW_R / 8; ++p) {
                const int jj = p * 8 + (lane >> 2);
                const long long t = t0 + jj;
                if (t >= 0 && c0 + cq < B) {
                    const int o = jj * CW_TC + cq;
                    const float4 v4 = *reinterpret_cast<const float4*>(rv + o);
                    const float4 n4 = *reinterpret_cast<const float4*>(rn + o);
                    const float4 r4 = *reinterpret_cast<const float4*>(rr + o);
                    const float4 d4 = has_done ? *reinterpret_cast<const float4*>(rd + o) : make_float4(0.f, 0.f, 0.f, 0.f);
                    const float4 t4 = has_traj ? *reinterpret_cast<const float4*>(rt + o) : d4;
                    float vv[4] = {v4.x, v4.y, v4.z, v4.w}, nn[4] = {n4.x, n4.y, n4.z, n4.w};
                    float rw[4] = {r4.x, r4.y, r4.z, r4.w}, dd[4] = {d4.x, d4.y, d4.z, d4.w};
                    float tt[4] = {t4.x, t4.y, t4.z, t4.w};
                    float de[4], fa[4];
                    bool changed = false;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if (has_done) {
                            changed |= (dd[k] != 0.f);
                            nn[k] = fmul(nn[k], fsub(1.f, dd[k]));
                        }
                        de[k] = fsub(fadd(rw[k], fmul(f.gamma, nn[k])), vv[k]);
                        fa[k] = fmul(f.gl, fsub(1.f, tt[k]));
                    }
                    *reinterpret_cast<float4*>(&ab[jj][cq]) = make_float4(de[0], de[1], de[2], de[3]);
                    *reinterpret_cast<float4*>(&fbuf[jj][cq]) = make_float4(fa[0], fa[1], fa[2], fa[3]);
                    if (changed && f.mask_inplace)
                        *reinterpret_cast<float4*>(f.next_value + t * B + c0 + cq) =
                            make_float4(nn[0], nn[1], nn[2], nn[3]);
                }
            }
            __syncwarp();
            // the raw slot has been read by every lane: refill it with the chunk two ahead
            if (item_valid(pf)) {
                issue_raw(pf, slot);
                item_next(pf);
            }
            cpa_commit();
            // ---- sequential scan, lane = column, newest time step first ---------------------------------------------------
            if (lane < CW_TC && c0 + lane < B) {
                if (t0 >= 0) {
                    float d[CW_R], g[CW_R];
#pragma unroll
                    for (int k = 0; k < CW_R; ++k) {
                        d[k] = ab[CW_R - 1 - k][lane];
                        g[k] = fbuf[CW_R - 1 - k][lane];
                    }
#pragma unroll
                    for (int k = 0; k < CW_R; ++k) {
                        carry = fadd(d[k], fmul(g[k], carry));
                        ab[CW_R - 1 - k][lane] = carry;
                    }
                } else {
                    for (int jj = CW_R - 1; jj >= 0 && t0 + jj >= 0; --jj) {
                        carry = fadd(ab[jj][lane], fmul(fbuf[jj][lane], carry));
                        ab[jj][lane] = carry;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&adv_ready[s]);
                if (j == 0) CW_TRACE(19);
            }
            // advantages -> HBM: R*4 = 64 float4, two per lane
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int p = lane + 32 * k;
                const int row = p >> 2, o = (p & 3) * 4;
                if (t0 + row >= 0 && c0 + o < B)
                    stg_stream4(reinterpret_cast<float4*>(a.adv_out + (t0 + row) * B + c0 + o),
                                *reinterpret_cast<const float4*>(&ab[row][o]));
            }
            if (++s == S) { s = 0; ph ^= 1; }
            item_next(it);
        }
        cpa_wait<0>();
    } else {
        // =============================================== consumers ========================================================
        PpoUpstream up{0.f, 0.f, 0.f, 0.f, 1.f / (float)a.S};
        if (GRADS) {
            up.g_pol = a.g_policy ? *a.g_policy : 0.f;
            up.g_val = a.g_value ? *a.g_value : 0.f;
            up.g_ent = a.g_entropy ? *a.g_entropy : 0.f;
            up.g_kl = (a.g_kl && has_pre) ? *a.g_kl : 0.f;
            if (a.g_used && blockIdx.x == 0 && tid == 0) {
                a.g_used[0] = up.g_pol; a.g_used[1] = up.g_val; a.g_used[2] = up.g_ent; a.g_used[3] = up.g_kl;
            }
        }
        const int jj = tid / CW_TC, c = tid % CW_TC;
        CwItem it = first;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            const long long c0 = it.tile * CW_TC;
            const long long t = T - (it.q + 1) * CW_R + jj;
            unsigned char* st = smem + s * L.stage_bytes;
            mbar_wait(&full[s], (uint32_t)ph);
            if (tid == 0 && j < 6) CW_TRACE(1 + 3 * j);
            mbar_wait(&adv_ready[s], (uint32_t)ph);
            if (tid == 0 && j < 6) CW_TRACE(2 + 3 * j);
            if (t >= 0 && c0 + c < B) {
                const long long g = t * B + c0 + c;  // global transition index
                float* grow = GRADS ? a.grad_logit + g * N : nullptr;
                float* gval = GRADS ? a.grad_value + g : nullptr;
                ppo_row_compute_to<NC, true, GRADS>(a, L, st, tid, N, advr[s][jj][c], grow, gval, up, acc);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&done[s]);
            if (tid == 0 && j < 6) CW_TRACE(3 + 3 * j);
            if (++s == S) { s = 0; ph ^= 1; }
            item_next(it);
        }
    }
    grid_store_partials<6, CW_THREADS>(acc, ws);  // summed by finalize_sums_kernel
}

static size_t cw_smem(int N, bool has_pre, bool has_w, int stages) {
    return (size_t)stages * cw_stage_bytes(N, has_pre, has_w) + 2 * CW_RAW_BYTES + CW_MAX_STAGES * CW_RAW_ARR + CW_RAW_ARR +
           3 * CW_MAX_STAGES * sizeof(uint64_t) + 32;
}

static int cw_pick_stages(const FusedArgs& f) {
    const PpoArgs& a = f.p;
    for (int s = CW_MAX_STAGES; s >= 2; --s)
        if (cw_smem(a.N, a.logit_pre != nullptr, a.weight != nullptr, s) <= 112 * 1024) return s;  // two CTAs per SM
    return 0;
}

bool colws_ok(const FusedArgs& f) {
    const PpoArgs& a = f.p;
    const bool al = aligned16(a.logit_new) && aligned16(a.logit_old) && (!a.logit_pre || aligned16(a.logit_pre)) &&
                    aligned16(a.action) && aligned16(a.value_new) && aligned16(a.value_old) && aligned16(a.ret) &&
                    (!a.weight || aligned16(a.weight)) && (!a.grad_logit || aligned16(a.grad_logit)) &&
                    (!a.grad_value || aligned16(a.grad_value)) && aligned16(f.value) && aligned16(f.next_value) &&
                    aligned16(f.reward) && aligned16(a.adv) && (!f.done || aligned16(f.done)) &&
                    (!f.traj || aligned16(f.traj));
    return al && a.N >= 1 && a.N <= 32 && f.T >= 1 && f.B >= 4 && (f.B % 4) == 0 && f.T * f.B == a.S &&
           cw_pick_stages(f) >= 2;
}

template <int NC, bool GRADS>
static int launch_ws(const FusedArgs& f, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    const PpoArgs& a = f.p;
    const int stages = cw_pick_stages(f);
    const size_t smem = cw_smem(a.N, a.logit_pre != nullptr, a.weight != nullptr, stages);
    constexpr auto kern = gae_ppo_ws_kernel<NC, GRADS>;
    int sm_count, per_sm;
    if (int rc = resident_ctas<kern>(CW_THREADS, smem, sm_count, per_sm)) return rc;
    const long long n_tiles = (f.B + CW_TC - 1) / CW_TC;
    long long grid = (long long)sm_count * per_sm;
    if (grid > n_tiles) grid = n_tiles;
    if (ws_bytes < WS_MIN_BYTES || !ws_partials_fit((long long)(grid * 6), ws_bytes))
        return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, CW_THREADS, smem, st, f, ws, stages)) return rc;
    FinalizeArgs fa = ppo_finalize_args(a.S, a.logit_pre != nullptr, (int)grid);
    // data-parallel training: the finalising threads stage the six scalars for the next step's kernel to publish (common.cuh)
    fa.x.mailboxes = f.x_mailboxes; fa.x.state = f.x_seq; fa.x.out_mean = f.x_out_mean; fa.x.rank = f.x_rank;
    fa.x.world = f.x_world;
    return launch_finalize(ws, out, fa, st);
}

template <bool GRADS>
static int dispatch_ws(const FusedArgs& f, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    return with_nc(f.p.N, [&](auto nc) { return launch_ws<nc, GRADS>(f, out, ws, ws_bytes, st); });
}

int launch_colws(const FusedArgs& f, bool grads, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    return grads ? dispatch_ws<true>(f, out, ws, ws_bytes, st) : dispatch_ws<false>(f, out, ws, ws_bytes, st);
}

}  // namespace b200rl
