// Column-tile learner step, warp-specialised: gae -> ppo_error (+ gradients) in ONE launch, no cross-CTA dependency, no
// CTA-wide barrier in the loop, every copy a plain 16-byte LDGSTS (cp.async) issued by a dedicated loader warp.
//
// Why a loader warp rather than every thread copying: with all threads copying and a __syncthreads per chunk, about half
// of the instructions go to copy addressing and the kernel is issue-bound.  Why per-lane LDGSTS rather than 2-D TMA boxes:
// the TMA unit's issue cost is per operation, and a column tile of the (T, B) tensors gives 64-byte box rows, 2 KB per
// operation (57 operations per tile), so the copies wait on the TMA unit instead.
//
// A CTA owns TC batch columns for ALL T (the recurrence of gae.py:65-69 runs along T only, ppo.py:77-140 is pointwise).
// Time is walked newest-first in chunks of R = 256 / TC steps (256 transitions).  Two geometries, chosen on the host from
// the SM count and B (cw_pick_tc):
//   TC = 32, R = 8    one CTA per SM, a ring of up to 8 stages; where 32-column tiles still give nearly every SM a tile
//                     (config D: B = 4096 -> 128 CTAs on an H100's 132 SMs, 16 chunks each).  Every (T, B) row segment is
//                     a full 128-byte line.
//   TC = 16, R = 16   two CTAs per SM, up to 4 stages each; every other shape (at config D: 256 CTAs, 8 chunks each).
// Warp roles (10 warps):
//   warp 8     loader: cp.async of the chunk's PPO inputs (logit_new | logit_old | action | value_new | value_old |
//              return_ [| weight | logit_pre]) into an S-stage ring (S = 8 / 4 at N = 6); completion arrives on the stage's
//              mbarrier (cp.async.mbarrier.arrive.noinc); a stage is refilled as soon as the consumers release it.
//   warp 9     scanner: own cp.async ring of the five GAE inputs (2 chunks deep; 4 with 32-column tiles, whose chunks
//              come twice as often); per chunk delta / f in the reference's operation order, the in-place next_value
//              mask (gae.py:61), the sequential scan A = delta + f*A (lane = column, separate round-to-nearest mul and
//              add: bit-identical to the torch loop); publishes the chunk's advantages in an S-slot shared-memory ring
//              (mbarrier) and writes them to HBM (16-byte coalesced).
//   warps 0-7  consumers: thread = transition; wait for "chunk landed" and "advantages ready", run ppo_row_compute_to (the
//              row code of ppo.cu) and store the gradient row (32-column tiles: through the row's logit_new slot, then
//              16-byte coalesced per warp) and the value gradient to HBM; arrive on "done".
// Rings run across tile boundaries (static tile -> CTA assignment: deterministic loss partial sums).
//
// Once the ring is primed the chunks stream at the rate HBM delivers them; what separates the kernel from the roofline
// is the time until the first chunk has landed and the tail (last chunk's math, store drain, partial sums,
// finalize_sums launch).  Measured with the stamps of tools/trace_col.py at config D on an H100 SXM (700 W, SM clock
// 1980 MHz): with 16 x 16 tiles the first chunk of a CTA landed 4.4 us (median) after griddepcontrol.wait -- the
// prologue requests four stages of all 256 CTAs, about 20 MB, before any has landed -- and the last CTA ended 24.1 us
// after it; with 32 x 8 tiles the first chunk lands after 2.6 us, a CTA then takes 1.2 - 1.3 us per chunk (3.9 MB over
// the grid) and 1.0 us from its last chunk landed to its end. That pace was the loader's while it copied with the flat
// loop (one loader warp per SM): on a 400 W card, whose SM clock drops under this load, the step stayed at 29.0 - 29.2
// us like the 16 x 16 tiles'; with warp copies and at most two stages in flight it is 27.1 - 27.2 us there.  Slower at
// config D on the H100: 6 stages instead of 8 (+0.4 us per step), requesting the first 2 or 4 chunks into L2
// (cp.async.bulk.prefetch) before griddepcontrol.wait (26.1 - 26.8 us and 27.9 us against 26.2; one chunk: no change).
// Storing the gradient rows straight from registers instead of through the stage: 26.2 - 26.7 us at config D, and 79 us
// against 52 at N = 18. Loader variants that were slower on B200: loop-invariant piece offsets in registers with one or
// two loader warps (the faster refill issues the ring of every CTA in one burst, which delays chunk 0 and costs DRAM
// efficiency), the same with a throttled prologue, no unrolling of the copy loop, 2 or 3 ring stages.
//
// Between two steps HBM idled: a CTA of the next step started 0.4 - 0.5 us (median over SMs) after the previous step's
// CTA on the same SM had ended (the 8-stage ring leaves no room for both), then waited for finalize_sums and the check
// launch and had its first chunk 5.8 - 6.5 us after that end.  A captured step that reads nothing those launches write
// therefore defers its griddepcontrol.wait (FusedArgs::defer_wait, decided on the host, common.cuh): its first chunk lands
// 2.4 - 5.4 us before the previous check has completed, and config D went from 25.8 to 24.2 us per step (H100 SXM, 700 W,
// 1980 MHz).  Slower: a 4-stage ring with __launch_bounds__(..., 2) (80 registers) in that mode, which lets the next
// step's CTA share the SM with the previous one on most SMs but streams slower: 27.7 us.
//
// Algorithmic traffic: 24 B (GAE) + 104 B (ppo_error forward + gradients, N = 6) = 128 B per transition, each byte once.
#include "../../include/b200rl.h"
#include "fused_args.cuh"

namespace b200rl {

constexpr int CW_CW = 8;                  // consumer warps
constexpr int CW_CT = CW_CW * 32;         // consumer threads = transitions per chunk
constexpr int CW_THREADS = CW_CT + 64;    // + loader warp + scanner warp
// Tile geometry (cw_pick_tc): TC = 16 columns x R = 16 steps per chunk, two CTAs per SM with up to 4 stages each, or
// TC = 32 columns x R = 8 steps, one CTA per SM with up to 8 stages.  A chunk is 256 transitions either way.
template <int TC> struct CwGeo {
    static constexpr int R = CW_CT / TC;                // time steps per chunk
    static constexpr int MAX_STAGES = TC == 32 ? 8 : 4;  // PPO ring stages
    static constexpr int CTAS_PER_SM = TC == 32 ? 1 : 2;
    static constexpr int PR = TC / 4;                   // 16-byte pieces per float row segment
    static constexpr int RAW_SLOTS = TC == 32 ? 4 : 2;  // scanner's ring of raw GAE chunks
};
// 32-column tiles: the loader copies every full stage with warp_copy_rows and keeps at most CW_AHEAD stages in flight
constexpr int CW_AHEAD = 2;  // 3, 4, 6: slower at config D on the H100 (tools/trace_col.py, bench.py)
constexpr int CW_RAW_ARR = CW_CT * 4;         // bytes of one raw GAE array chunk
constexpr int CW_RAW_BYTES = 5 * CW_RAW_ARR;  // value | next_value | reward | done | traj_flag

// B200RL_FUSED_TRACE=1: %globaltimer stamps, 64 per CTA (tools/trace_col.py).  Slots 0-7 frame the CTA: 0 start, 1 the
// previous launches' results visible (after griddepcontrol.wait), 2 first chunk's advantages published, 3 / 4 / 5 the
// last chunk landed / advantages ready / computed, 6 end (partial sums stored), 7 the number of chunks (low 32 bits) and
// the SM the CTA ran on (high 32 bits).  Chunk j < CW_TRACE_CHUNKS: 8 + 4j landed, 9 + 4j advantages ready, 10 + 4j
// computed, 11 + 4j its stage issued by the loader.  Slot 60: chunk 0 landed as the loader sees it (32-column tiles; in
// a deferred launch that can be before the consumers' wait).
constexpr int CW_TRACE_CHUNKS = 13;
#define CW_TRACE(slot)                                                                                   \
    do {                                                                                                 \
        if (f.trace) reinterpret_cast<unsigned long long*>(ws + 65536)[blockIdx.x * 64 + (slot)] = gtimer(); \
    } while (0)

struct CwItem {
    long long tile;
    long long q;  // chunk from the top of the trajectory: time steps [T - (q+1)R, T - qR)
};

__host__ __device__ inline int cw_stage_bytes(int N, bool has_pre, bool has_w) {
    return (CW_CT * ((has_pre ? 3 : 2) * N * 4 + 8 + 12 + (has_w ? 4 : 0)) + 127) & ~127;
}

template <int NC, bool GRADS, int TC>
__global__ void __launch_bounds__(CW_THREADS, CwGeo<TC>::CTAS_PER_SM) gae_ppo_ws_kernel(FusedArgs f, float* ws, int n_stages) {
    constexpr int CW_R = CwGeo<TC>::R, CW_MAX_STAGES = CwGeo<TC>::MAX_STAGES, PR = CwGeo<TC>::PR;
    constexpr int RAWS = CwGeo<TC>::RAW_SLOTS;
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
    unsigned char* raw = smem + S * L.stage_bytes;                                            // [RAWS][5][R][TC]
    auto advr = reinterpret_cast<float (*)[CW_R][TC]>(raw + RAWS * CW_RAW_BYTES);            // [S][R][TC]
    auto fbuf = reinterpret_cast<float (*)[TC]>(reinterpret_cast<unsigned char*>(advr) + CW_MAX_STAGES * CW_RAW_ARR);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(fbuf) + CW_RAW_ARR);
    uint64_t* full = bars;                           // [S] PPO chunk landed (32 loader-lane arrivals)
    uint64_t* done = bars + CW_MAX_STAGES;           // [S] consumers finished the chunk (CW_CW arrivals)
    uint64_t* adv_ready = bars + 2 * CW_MAX_STAGES;  // [S] advantages of the chunk are in advr[s]

    const long long T = f.T, B = f.B;
    const long long n_tiles = (B + TC - 1) / TC;
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
    // PDL.  The wait for the previous launches' results comes after the barrier set-up (nothing before it touches global
    // memory except the optional trace stamp), and the next launch may start only after it: so when a later column kernel
    // starts, everything enqueued before this one has completed.  Deferred (f.defer_wait, common.cuh): only the warps that
    // write wait -- the loader streams the chunks in while the previous step's finalize and check launches finish.
    auto dep_wait = [] {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    };
    if (!f.defer_wait) dep_wait();
    __syncthreads();
    if (tid == 0 && !f.defer_wait) CW_TRACE(1);
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
            const int P = TC * esz / 16, Pv = W * esz / 16;
            const unsigned char* g = reinterpret_cast<const unsigned char*>(src) + (t0 * B + c0) * esz;
            const long long rstride = B * esz;
            const int n = CW_R * P;
#pragma unroll 4
            for (int p = lane; p < n; p += 32) {
                const int row = p / P, o = p - row * P;
                if (row >= jmin && o < Pv) cpa16(dst + p * 16, g + row * rstride + o * 16);
            }
        };
        // 16-column tiles: the FIRST stage of a CTA uses lane-owns-a-piece-column copies (common.cuh warp_copy_rows, ~3
        // instructions per copy), every later one the flat loop (~35 instructions per copy).  Two CTAs per SM stream at the
        // HBM rate in steady state, so a faster loader buys nothing there -- issued in bursts the copies only deepen the
        // queues in front of everybody's next chunk -- but the first stage is pure latency: the flat loop's address
        // arithmetic runs before the first byte is requested.
        // 32-column tiles (one CTA, so one loader warp per SM): the flat loop takes ~1.3 us to issue a stage at 1980 MHz,
        // as long as HBM takes to deliver one, and longer at the lower clock of a power-capped card -- the loader, not HBM,
        // set the pace.  So every full stage uses warp_copy_rows, and the loader keeps at most CW_AHEAD stages in flight:
        // copying the whole 8-stage ring in one burst made the step 30.1 us against 26.2 (chunk 0 waits behind it).
        CwItem it = first;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            if (j >= S) mbar_wait(&done[s], (uint32_t)(ph ^ 1));
            if (TC == 32 && j >= CW_AHEAD) {  // chunk j - CW_AHEAD has landed
                const int jb = j - CW_AHEAD;
                mbar_wait(&full[jb % S], (uint32_t)((jb / S) & 1));
                if (jb == 0 && lane == 0) CW_TRACE(60);
            }
            const long long c0 = it.tile * TC;
            const long long t0 = T - (it.q + 1) * CW_R;
            const int jmin = t0 < 0 ? (int)-t0 : 0;
            const int W = (int)((B - c0) < TC ? (B - c0) : TC);
            unsigned char* st = smem + s * L.stage_bytes;
            if (jmin == 0 && W == TC && (TC == 32 || j == 0)) {
                // full chunk of a full tile, 16 columns: a row segment is TC * esz / 16 = esz pieces (4 N | 8 | 4).  Logits
                // and actions go in 8-piece groups (a lane group covers one full 128-byte line per row: the 4-piece grouping
                // doubles the number of L2 requests, which makes it slower than the flat loop); the float tensors have
                // 64-byte rows.
                const uint32_t sb = smem_u32(st);
                const long long e0 = t0 * B + c0;
                const long long ls = B * N * 4;
                if constexpr (TC == 32) {
                    // 32-column rows: 8 lanes cover one 128-byte line of every tensor, N lines per logit row segment
                    warp_copy_rows<8, CW_R, NC>(sb, a.logit_new + e0 * N, ls, N, lane);
                    warp_copy_rows<8, CW_R, NC>(sb + L.off_old, a.logit_old + e0 * N, ls, N, lane);
                    if (has_pre) warp_copy_rows<8, CW_R, NC>(sb + L.off_pre, a.logit_pre + e0 * N, ls, N, lane);
                    warp_copy_rows<8, CW_R, 2>(sb + L.off_act, a.action + e0, B * 8, 2, lane);
                } else if (N & 1) {
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
                warp_copy_rows<PR, CW_R, 1>(sb + L.off_vn, a.value_new + e0, B * 4, 1, lane);
                warp_copy_rows<PR, CW_R, 1>(sb + L.off_vo, a.value_old + e0, B * 4, 1, lane);
                warp_copy_rows<PR, CW_R, 1>(sb + L.off_ret, a.ret + e0, B * 4, 1, lane);
                if (has_w) warp_copy_rows<PR, CW_R, 1>(sb + L.off_w, a.weight + e0, B * 4, 1, lane);
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
            if (f.trace && lane == 0 && j < CW_TRACE_CHUNKS) CW_TRACE(11 + 4 * j);
            if (++s == S) { s = 0; ph ^= 1; }
            item_next(it);
        }
    } else if (wid == CW_CW + 1) {
        // =============================================== scanner ==========================================================
        auto issue_raw = [&](const CwItem& it, int slot) {
            const long long c0 = it.tile * TC;
            const long long t0 = T - (it.q + 1) * CW_R;
            const int W = (int)((B - c0) < TC ? (B - c0) : TC);
            unsigned char* dst = raw + slot * CW_RAW_BYTES;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int p = lane + 32 * k;  // R * TC / 4 = 64 pieces per array
                const int row = p / PR, o = p % PR;
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
        for (int k = 0; k < RAWS; ++k) {
            if (item_valid(pf)) {
                issue_raw(pf, k);
                item_next(pf);
            }
            cpa_commit();
        }
        if (f.defer_wait) {  // before the first store (the in-place next_value mask, the advantages)
            dep_wait();
            if (lane == 0) CW_TRACE(1);
        }
        float carry = 0.f;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            const long long c0 = it.tile * TC;
            const long long t0 = T - (it.q + 1) * CW_R;
            const int slot = j % RAWS;
            if (it.q == 0) carry = 0.f;
            cpa_wait<RAWS - 1>();
            __syncwarp();
            if (j >= S) mbar_wait(&done[s], (uint32_t)(ph ^ 1));  // the consumers are through the chunk that used advr[s]
            float (*ab)[TC] = advr[s];
            const float* rv = reinterpret_cast<const float*>(raw + slot * CW_RAW_BYTES);
            const float* rn = rv + CW_R * TC;
            const float* rr = rn + CW_R * TC;
            const float* rd = rr + CW_R * TC;
            const float* rt = rd + CW_R * TC;
            const int cq = (lane % PR) * 4;
#pragma unroll
            for (int p = 0; p < CW_R * PR / 32; ++p) {
                const int jj = p * (32 / PR) + lane / PR;
                const long long t = t0 + jj;
                if (t >= 0 && c0 + cq < B) {
                    const int o = jj * TC + cq;
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
            // the raw slot has been read by every lane: refill it with the chunk RAWS ahead
            if (item_valid(pf)) {
                issue_raw(pf, slot);
                item_next(pf);
            }
            cpa_commit();
            // ---- sequential scan, lane = column, newest time step first ---------------------------------------------------
            if (lane < TC && c0 + lane < B) {
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
                if (j == 0) CW_TRACE(2);
            }
            // advantages -> HBM: R * TC / 4 = 64 float4, two per lane
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int p = lane + 32 * k;
                const int row = p / PR, o = (p % PR) * 4;
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
        if (f.defer_wait) dep_wait();  // before the upstream-gradient record and every gradient store
        float g[4] = {0.f, 0.f, 0.f, 0.f};
        if (GRADS) upstream<4>(a.rec, false, ppo_owned(a), g);  // a forward launch: records `used`, never skips
        const PpoUpstream up{g[0], g[1], g[2], g[3], 1.f / (float)a.S};
        // trace: chunk j's stamp k (0 landed, 1 advantages ready, 2 computed); slots 3-5 are overwritten by every chunk, so
        // the last chunk's remain
        auto stamp_chunk = [&](int j, int k) {
            if (f.trace && tid == 0) {
                unsigned long long* tr = reinterpret_cast<unsigned long long*>(ws + 65536) + blockIdx.x * 64;
                const unsigned long long now = gtimer();
                tr[3 + k] = now;
                if (j < CW_TRACE_CHUNKS) tr[8 + 4 * j + k] = now;
                if (k == 2) tr[7] = (unsigned long long)smid() << 32 | (unsigned long long)(j + 1);
            }
        };
        const int jj = tid / TC, c = tid % TC;
        CwItem it = first;
        int s = 0, ph = 0;
        for (int j = 0; item_valid(it); ++j) {
            const long long c0 = it.tile * TC;
            const long long t = T - (it.q + 1) * CW_R + jj;
            unsigned char* st = smem + s * L.stage_bytes;
            mbar_wait(&full[s], (uint32_t)ph);
            stamp_chunk(j, 0);
            mbar_wait(&adv_ready[s], (uint32_t)ph);
            stamp_chunk(j, 1);
            // 32-column tiles: a warp is one time step of 32 consecutive transitions, so its gradient rows are one contiguous
            // 128*N-byte span in HBM.  They go to the rows' own logit_new slots in the stage first and leave as 16-byte
            // coalesced stores (full lines instead of 8 bytes into each of 24 sectors per store instruction at N = 6).
            const bool stage_grads = GRADS && TC == 32 && t >= 0 && c0 + TC <= B;  // warp-uniform
            if (t >= 0 && c0 + c < B) {
                const long long g = t * B + c0 + c;  // global transition index
                float* grow = GRADS ? (stage_grads ? reinterpret_cast<float*>(st) + tid * N : a.grad_logit + g * N)
                                    : nullptr;
                float* gval = GRADS ? a.grad_value + g : nullptr;
                ppo_row_compute_to<NC, true, GRADS>(a, L, st, tid, N, advr[s][jj][c], grow, gval, up, acc);
            }
            if (stage_grads) {
                __syncwarp();
                const float4* src = reinterpret_cast<const float4*>(st) + wid * 8 * N;  // 32 rows of N floats
                float4* dst = reinterpret_cast<float4*>(a.grad_logit + (t * B + c0) * N);
                for (int k = lane; k < 8 * N; k += 32) stg_stream4(dst + k, src[k]);
            }
            __syncwarp();  // every lane's reads of the stage precede the release
            if (lane == 0) mbar_arrive(&done[s]);
            stamp_chunk(j, 2);
            if (++s == S) { s = 0; ph ^= 1; }
            item_next(it);
        }
    }
    grid_store_partials<6, CW_THREADS>(acc, ws);  // summed by finalize_sums_kernel
    if (tid == 0) CW_TRACE(6);
}

template <int TC>
static size_t cw_smem(int N, bool has_pre, bool has_w, int stages) {
    constexpr int MS = CwGeo<TC>::MAX_STAGES;
    return (size_t)stages * cw_stage_bytes(N, has_pre, has_w) + CwGeo<TC>::RAW_SLOTS * CW_RAW_BYTES + MS * CW_RAW_ARR +
           CW_RAW_ARR + 3 * MS * sizeof(uint64_t) + 32;
}

// deepest PPO ring that keeps CwGeo<TC>::CTAS_PER_SM CTAs resident per SM (0: not even two stages)
template <int TC>
static int cw_stages(const FusedArgs& f) {
    const PpoArgs& a = f.p;
    const size_t limit = CwGeo<TC>::CTAS_PER_SM == 2 ? 112 * 1024 : 227 * 1024;
    for (int s = CwGeo<TC>::MAX_STAGES; s >= 2; --s)
        if (cw_smem<TC>(a.N, a.logit_pre != nullptr, a.weight != nullptr, s) <= limit) return s;
    return 0;
}

// Tile width for this shape on a device with `sm_count` SMs.  32-column tiles make every (T, B) row segment a full
// 128-byte line and give each CTA twice as many chunks (one CTA per SM, a ring of up to 8 stages).  They are taken when
// they keep at least as many stages in flight per SM, leave at most 1/16 of the SMs without a tile, and give the busiest
// SM no more columns than 16-column tiles (two CTAs per SM) do: at B = 4096 on 132 SMs, 128 CTAs of 32 columns against
// 256 CTAs of 16, 32 columns on the busiest SM either way.
static int cw_pick_tc(const FusedArgs& f, int sm_count) {
    const int s16 = cw_stages<16>(f), s32 = cw_stages<32>(f);
    if (s32 < 2 * s16) return 16;
    const long long n16 = (f.B + 15) / 16, n32 = (f.B + 31) / 32;
    if (n32 < sm_count - sm_count / 16) return 16;
    const long long cols16 = 16 * ((n16 + sm_count - 1) / sm_count), cols32 = 32 * ((n32 + sm_count - 1) / sm_count);
    return cols32 <= cols16 ? 32 : 16;
}

bool colws_ok(const FusedArgs& f) {
    const PpoArgs& a = f.p;
    const bool al = aligned16(a.logit_new) && aligned16(a.logit_old) && (!a.logit_pre || aligned16(a.logit_pre)) &&
                    aligned16(a.action) && aligned16(a.value_new) && aligned16(a.value_old) && aligned16(a.ret) &&
                    (!a.weight || aligned16(a.weight)) && (!a.grad_logit || aligned16(a.grad_logit)) &&
                    (!a.grad_value || aligned16(a.grad_value)) && aligned16(f.value) && aligned16(f.next_value) &&
                    aligned16(f.reward) && aligned16(a.adv) && (!f.done || aligned16(f.done)) &&
                    (!f.traj || aligned16(f.traj));
    // the 16-column geometry takes every shape; the 32-column one only replaces it where cw_pick_tc says so
    return al && a.N >= 1 && a.N <= 32 && f.T >= 1 && f.B >= 4 && (f.B % 4) == 0 && f.T * f.B == a.S &&
           cw_stages<16>(f) >= 2;
}

// the bytes a deferred launch reads before its dependency wait: the loader's and the scanner's inputs
static int cw_early_reads(const FusedArgs& f, ByteSpan* r) {
    const PpoArgs& a = f.p;
    const long long S = a.S, L = S * a.N * 4, F = S * 4;
    const ByteSpan s[] = {byte_span(a.logit_new, L), byte_span(a.logit_old, L), byte_span(a.logit_pre, L),
                          byte_span(a.action, S * 8),   byte_span(a.value_new, F), byte_span(a.value_old, F),
                          byte_span(a.ret, F),          byte_span(a.weight, F),    byte_span(f.value, F),
                          byte_span(f.next_value, F),   byte_span(f.reward, F),    byte_span(f.done, F),
                          byte_span(f.traj, F)};
    for (const ByteSpan& x : s) *r++ = x;
    return (int)(sizeof(s) / sizeof(s[0]));
}

// the bytes the column kernel and its finalize launch may write
static int cw_writes(const FusedArgs& f, float* out, float* ws, size_t ws_bytes, ByteSpan* w) {
    const PpoArgs& a = f.p;
    const long long S = a.S, F = S * 4;
    const ByteSpan s[] = {byte_span(a.adv_out, F),
                          byte_span(a.grad_logit, S * a.N * 4),
                          byte_span(a.grad_value, F),
                          byte_span(f.mask_inplace ? f.next_value : nullptr, F),
                          byte_span(a.rec.used, 4 * sizeof(float)),
                          byte_span(ws, (long long)ws_bytes),
                          byte_span(out, 8 * sizeof(float)),
                          byte_span(f.x_seq, 24 * sizeof(unsigned int)),
                          byte_span(f.x_out_mean, 16 * sizeof(float))};
    for (const ByteSpan& x : s) *w++ = x;
    return (int)(sizeof(s) / sizeof(s[0]));
}

template <int NC, bool GRADS, int TC>
static int launch_ws(const FusedArgs& f_in, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    FusedArgs f = f_in;
    const PpoArgs& a = f.p;
    // captured straight behind the previous step's launches and reading nothing they write: defer the wait (common.cuh)
    const ChainPoint at = capture_now(st);
    ByteSpan span[16];
    f.defer_wait = !f.x_mailboxes && chain_may_defer(st, at, span, cw_early_reads(f, span));
    const int stages = cw_stages<TC>(f);
    const size_t smem = cw_smem<TC>(a.N, a.logit_pre != nullptr, a.weight != nullptr, stages);
    constexpr auto kern = gae_ppo_ws_kernel<NC, GRADS, TC>;
    int sm_count, per_sm;
    if (int rc = resident_ctas<kern>(CW_THREADS, smem, sm_count, per_sm)) return rc;
    if (per_sm > CwGeo<TC>::CTAS_PER_SM) per_sm = CwGeo<TC>::CTAS_PER_SM;
    const long long n_tiles = (f.B + TC - 1) / TC;
    long long grid = (long long)sm_count * per_sm;
    if (grid > n_tiles) grid = n_tiles;
    if (ws_bytes < WS_MIN_BYTES || !ws_partials_fit((long long)(grid * 6), ws_bytes))
        return B200RL_ERR_WORKSPACE;
    if (int rc = launch_k(kern, (int)grid, CW_THREADS, smem, st, f, ws, stages)) return rc;
    FinalizeArgs fa = ppo_finalize_args(a.S, a.logit_pre != nullptr, (int)grid);
    // data-parallel training: the finalising threads stage the six scalars for the next step's kernel to publish (common.cuh)
    fa.x.mailboxes = f.x_mailboxes; fa.x.state = f.x_seq; fa.x.out_mean = f.x_out_mean; fa.x.rank = f.x_rank;
    fa.x.world = f.x_world;
    if (int rc = launch_finalize(ws, out, fa, st)) return rc;
    chain_report(st, at, true, span, cw_writes(f, out, ws, ws_bytes, span));
    return B200RL_OK;
}

template <bool GRADS>
static int dispatch_ws(const FusedArgs& f, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    int sm_count = 0;
    if (int rc = sm_count_of(sm_count)) return rc;
    const int tc = cw_pick_tc(f, sm_count);
    return with_nc(f.p.N, [&](auto nc) {
        return tc == 32 ? launch_ws<nc, GRADS, 32>(f, out, ws, ws_bytes, st) : launch_ws<nc, GRADS, 16>(f, out, ws, ws_bytes, st);
    });
}

int launch_colws(const FusedArgs& f, bool grads, float* out, float* ws, size_t ws_bytes, cudaStream_t st) {
    return grads ? dispatch_ws<true>(f, out, ws, ws_bytes, st) : dispatch_ws<false>(f, out, ws, ws_bytes, st);
}

}  // namespace b200rl
