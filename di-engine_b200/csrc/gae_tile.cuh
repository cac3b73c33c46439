#pragma once
// Shared device code of the GAE column-tile scan (gae.cu) and the fused one-pass learner step (fused.cu).
#include "common.cuh"

namespace b200rl {

// named barriers with immediate ids (a register id would make ptxas reserve all 16 hardware barriers per CTA)
template <int ID, int COUNT>
__device__ __forceinline__ void named_bar_sync() {
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(COUNT) : "memory");
}
template <int ID, int COUNT>
__device__ __forceinline__ void named_bar_arrive() {
    asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(COUNT) : "memory");
}
template <int COUNT>
__device__ __forceinline__ void chunk_arrive(int k) {
    if (k == 0) named_bar_arrive<1, COUNT>();
    else if (k == 1) named_bar_arrive<2, COUNT>();
    else if (k == 2) named_bar_arrive<3, COUNT>();
    else named_bar_arrive<4, COUNT>();
}
// chunk-scanned barriers 5..8: the scan warp (32) arrives, one storer warp (32) waits
__device__ __forceinline__ void scanned_arrive(int k) {
    if (k == 0) named_bar_arrive<5, 64>();
    else if (k == 1) named_bar_arrive<6, 64>();
    else if (k == 2) named_bar_arrive<7, 64>();
    else named_bar_arrive<8, 64>();
}
__device__ __forceinline__ void scanned_wait(int k) {
    if (k == 0) named_bar_sync<5, 64>();
    else if (k == 1) named_bar_sync<6, 64>();
    else if (k == 2) named_bar_sync<7, 64>();
    else named_bar_sync<8, 64>();
}
template <int COUNT>
__device__ __forceinline__ void chunk_wait(int k) {
    if (k == 0) named_bar_sync<1, COUNT>();
    else if (k == 1) named_bar_sync<2, COUNT>();
    else if (k == 2) named_bar_sync<3, COUNT>();
    else named_bar_sync<4, COUNT>();
}

constexpr int GAE_CH = 32;      // rows per chunk (one named barrier per chunk)
constexpr int GAE_NCHUNK = 4;   // chunks per slab of T
constexpr int GAE_SLAB = GAE_CH * GAE_NCHUNK;

// Device body shared by gae_ws_kernel (gae.cu) and the fused learner step (fused.cu): one column tile [c0, c0+TC) for
// all T.  Thread roles: threadIdx.x < 32 scan warp, the next TC/4 warps loaders (and, once their loads are consumed,
// storers of the finished chunks).  `on_chunk_done(global_chunk, any)` is called by a whole storer warp after it has
// stored the adv rows of a 32-row chunk (newest chunk = 0).
template <int TC, bool VEC, class OnChunk>
__device__ __forceinline__ void gae_tile_body(
    const float* __restrict__ value, float* __restrict__ next_value, const float* __restrict__ reward,
    const float* __restrict__ done, const float* __restrict__ traj, float* __restrict__ adv, long long T,
    long long C, long long A, float gamma, float gl, int mask_inplace, long long c0,
    float (*s_d)[GAE_CH][TC], float (*s_f)[GAE_CH][TC], OnChunk on_chunk_done, float vscale = 0.f) {
    constexpr int NL = (TC / 4) * 32;  // loader threads
    constexpr int NTHREADS = NL + 32;
    const long long Caux = C / A;
    const bool is_scan = threadIdx.x < 32;
    const int ltid = threadIdx.x - 32;  // loader thread index
    float carry = 0.f;                  // scan lanes
    for (long long hi = T; hi > 0; hi -= GAE_SLAB) {
        const long long lo = hi > GAE_SLAB ? hi - GAE_SLAB : 0;
        const int rows = (int)(hi - lo);
        // chunk k covers slab rows [rlo_k, rhi_k), k = 0 is the newest (processed first)
        if (!is_scan) {
            if (VEC) {
                constexpr int TPR = TC / 4;  // NL / TPR == 32 rows per pass == one chunk
                const int cq = (ltid % TPR) * 4;
                const int rr = ltid / TPR;   // row inside the chunk, counted from the chunk's top (newest) row
                const long long c = c0 + cq;
                const bool col_ok = c < C;
                // software pipeline, GAE_DEPTH chunks in flight per thread (newest first): the loads of chunk k+DEPTH are
                // issued only when chunk k has been consumed, so chunk 0 of EVERY column tile arrives before anybody's
                // chunk 2 -- the scan (and, in the fused kernel, the PPO tiles of the newest time steps) can start after a
                // quarter of the bytes instead of all of them
                constexpr int DEPTH = 2;
                float4 v[DEPTH], nv[DEPTH], rw[DEPTH], dn[DEPTH], tf[DEPTH];
                auto issue = [&](int k, int b) {
                    const int r = rows - 1 - k * GAE_CH - rr;  // slab row of this thread in chunk k
                    if (r >= 0 && col_ok) {
                        const long long off = (lo + r) * C + c;
                        v[b] = ldg_stream4(reinterpret_cast<const float4*>(value + off));
                        nv[b] = ldg_stream4(reinterpret_cast<const float4*>(next_value + off));
                        rw[b] = ldg_stream4(reinterpret_cast<const float4*>(reward + off));
                        dn[b] = done ? ldg_stream4(reinterpret_cast<const float4*>(done + off))
                                     : make_float4(0.f, 0.f, 0.f, 0.f);
                        tf[b] = traj ? ldg_stream4(reinterpret_cast<const float4*>(traj + off)) : dn[b];
                    }
                };
#pragma unroll
                for (int k = 0; k < DEPTH; ++k) issue(k, k);
#pragma unroll
                for (int k = 0; k < GAE_NCHUNK; ++k) {
                    const int b = k % DEPTH;
                    const int r = rows - 1 - k * GAE_CH - rr;
                    if (r >= 0 && col_ok) {
                        float vv[4] = {v[b].x, v[b].y, v[b].z, v[b].w}, nn[4] = {nv[b].x, nv[b].y, nv[b].z, nv[b].w};
                        float rw4[4] = {rw[b].x, rw[b].y, rw[b].z, rw[b].w};
                        float dd[4] = {dn[b].x, dn[b].y, dn[b].z, dn[b].w};
                        float tt[4] = {tf[b].x, tf[b].y, tf[b].z, tf[b].w};
                        float de[4], fa[4];
                        bool changed = false;
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            if (vscale != 0.f) {  // value_norm: value *= std; next_value *= std (ding/policy/ppo.py:276-278)
                                vv[q] = fmul(vv[q], vscale);
                                nn[q] = fmul(nn[q], vscale);
                            }
                            if (done) {
                                changed |= (dd[q] != 0.f);
                                nn[q] = fmul(nn[q], fsub(1.f, dd[q]));
                            }
                            de[q] = fsub(fadd(rw4[q], fmul(gamma, nn[q])), vv[q]);
                            fa[q] = fmul(gl, fsub(1.f, tt[q]));
                        }
                        *reinterpret_cast<float4*>(&s_d[k][rr][cq]) = make_float4(de[0], de[1], de[2], de[3]);
                        *reinterpret_cast<float4*>(&s_f[k][rr][cq]) = make_float4(fa[0], fa[1], fa[2], fa[3]);
                        if (changed && mask_inplace)
                            *reinterpret_cast<float4*>(next_value + (lo + r) * C + c) =
                                make_float4(nn[0], nn[1], nn[2], nn[3]);
                    }
                    chunk_arrive<NTHREADS>(k);
                    if (k + DEPTH < GAE_NCHUNK) issue(k + DEPTH, b);
                }
            } else {
#pragma unroll
                for (int k = 0; k < GAE_NCHUNK; ++k) {
                    const int rtop = rows - 1 - k * GAE_CH;  // newest slab row of chunk k
                    for (int i = ltid; i < GAE_CH * TC; i += NL) {
                        const int rr = i / TC, cc = i % TC;
                        const int r = rtop - rr;
                        const long long c = c0 + cc;
                        if (r >= 0 && c < C) {
                            const long long off = (lo + r) * C + c;
                            const long long aoff = (lo + r) * Caux + c / A;
                            float nvv = next_value[off];
                            if (vscale != 0.f) nvv = fmul(nvv, vscale);
                            const float dnn = done ? done[aoff] : 0.f;
                            const float tff = traj ? traj[aoff] : dnn;
                            if (done) {
                                const float mm = fmul(nvv, fsub(1.f, dnn));
                                if (mask_inplace && dnn != 0.f) next_value[off] = mm;
                                nvv = mm;
                            }
                            const float vvv = vscale != 0.f ? fmul(value[off], vscale) : value[off];
                            s_d[k][rr][cc] = fsub(fadd(reward[aoff], fmul(gamma, nvv)), vvv);
                            s_f[k][rr][cc] = fmul(gl, fsub(1.f, tff));
                        }
                    }
                    chunk_arrive<NTHREADS>(k);
                }
            }
        } else {
            const int cc = threadIdx.x;
            const bool lane_ok = cc < TC && c0 + cc < C;
#pragma unroll 1
            for (int k = 0; k < GAE_NCHUNK; ++k) {
                chunk_wait<NTHREADS>(k);
                const int rtop = rows - 1 - k * GAE_CH;
                if (lane_ok && rtop >= 0) {
                    if (rtop >= GAE_CH - 1) {  // full chunk: registers first, then the dependent chain
                        float d[GAE_CH], f[GAE_CH];
#pragma unroll
                        for (int j = 0; j < GAE_CH; ++j) {
                            d[j] = s_d[k][j][cc];
                            f[j] = s_f[k][j][cc];
                        }
#pragma unroll
                        for (int j = 0; j < GAE_CH; ++j) {
                            carry = fadd(d[j], fmul(f[j], carry));
                            s_d[k][j][cc] = carry;
                        }
                    } else {
                        for (int j = 0; j <= rtop; ++j) {
                            carry = fadd(s_d[k][j][cc], fmul(s_f[k][j][cc], carry));
                            s_d[k][j][cc] = carry;
                        }
                    }
                }
                scanned_arrive(k);  // hand the finished chunk to its storer warp and go straight on to the next chunk
            }
        }
        // ---- storer: loader warp (k mod #loader warps) writes chunk k to HBM, coalesced, off the scan's critical path ----
        if (!is_scan) {
            constexpr int NLW = NL / 32;
            const int lw = ltid >> 5, ll = ltid & 31;
#pragma unroll 1
            for (int k = 0; k < GAE_NCHUNK; ++k) {
                if (k % NLW != lw) continue;
                scanned_wait(k);
                const int rtop = rows - 1 - k * GAE_CH;
                if (VEC) {
                    constexpr int TPR = TC / 4;
                    for (int i = ll; i < GAE_CH * TPR; i += 32) {
                        const int rr = i / TPR, cq = (i % TPR) * 4;
                        const int r = rtop - rr;
                        if (r >= 0 && c0 + cq < C) {
                            const float4 a4 = *reinterpret_cast<const float4*>(&s_d[k][rr][cq]);
                            stg_stream4(reinterpret_cast<float4*>(adv + (lo + r) * C + c0 + cq), a4);
                        }
                    }
                } else {
                    for (int i = ll; i < GAE_CH * TC; i += 32) {
                        const int rr = i / TC, cc = i % TC;
                        const int r = rtop - rr;
                        if (r >= 0 && c0 + cc < C) adv[(lo + r) * C + c0 + cc] = s_d[k][rr][cc];
                    }
                }
                on_chunk_done((T - hi) / GAE_CH + k, rtop >= 0);  // called by the whole storer warp
            }
        }
        if (lo > 0) __syncthreads();  // the next slab reuses the chunk buffers
    }
}

}  // namespace b200rl
