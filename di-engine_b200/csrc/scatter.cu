// ScatterConnection (ding/torch_utils/network/scatter_connection.py:59-121): entity rows x[b, m, :] scattered into a
// (B, N, H*W) map at the flat index idx[b, m] = col[b, m] + row[b, m] * W, and the gather that is its gradient.
//
// Forward, one launch and no memset: a CTA owns a tile of SC_NT features x SC_CELLS cells of one b.  It reads b's M
// indices (an L2-resident 16*M bytes), orders the entities of its cell tile by (cell, m) with a counting sort in shared
// memory, then one warp per cell adds the rows x[b, m, n-tile] (lane = n, coalesced) in ascending m -- the order of the
// CPU scatter_add_ -- or keeps the row of the largest m ('cover', the CPU scatter_'s result).  The finished tile is written
// once, coalesced along cells, zeros included.  No atomics touch a value, so every run gives the same bits.
//
// Backward, one launch, d x[b, m, n] = g[b, n, idx[b, m]] (zero for an out-of-range index), in one of two forms chosen
// from the shapes: the tile kernel stages g's (feature x cell) tiles through shared memory with coalesced reads when the
// entities are dense enough that gathering would fetch as many sectors as reading all of g (M * 8 >= H*W, 8 floats per
// 32-byte sector); otherwise the gather kernel reads only the B*M*N values it needs.
#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {
namespace {
constexpr int SC_THREADS = 256;
constexpr int SC_WARPS = SC_THREADS / 32;
constexpr int SC_CELLS = 128;             // cells per tile
constexpr int SC_NT = 32;                 // features per tile: lane = n
constexpr int SC_PITCH = SC_CELLS + 1;    // a column (fixed cell, lane = n) and a row (fixed n, lane = cell) are both conflict-free
constexpr int SC_CHUNK = 512;             // entities sorted per pass
constexpr int SC_SEG = SC_CHUNK / SC_WARPS;  // each warp counts and places a contiguous segment of the chunk
constexpr int SC_SECTOR_FLOATS = 8;       // floats per 32-byte sector: the dense / gather crossover of the backward
constexpr unsigned FULL = 0xffffffffu;

struct ScatterIndex {
    const long long* row;  // multiplied by W: location[..., 0] (forward), coord_x (xy_forward)
    long long row_sb, row_sm;
    const long long* col;  // location[..., 1], coord_y
    long long col_sb, col_sm;
    long long W, HW;
};

// int64 arithmetic that wraps as torch's does; only 0 <= idx < HW is a valid index
__device__ __forceinline__ long long flat_index(const ScatterIndex& ix, long long b, long long m) {
    const unsigned long long r = (unsigned long long)__ldg(ix.row + b * ix.row_sb + m * ix.row_sm);
    const unsigned long long c = (unsigned long long)__ldg(ix.col + b * ix.col_sb + m * ix.col_sm);
    return (long long)(c + r * (unsigned long long)ix.W);
}

// six resident CTAs (151 KB of shared memory) leave ptxas 40 registers: the cover variant spills without the bound
template <bool COVER>
__global__ void __launch_bounds__(SC_THREADS, 6) scatter_fwd_kernel(const float* __restrict__ x, long long x_sb, long long x_sm,
                                                                 long long x_sn, ScatterIndex ix, int M, int N, int n_ctiles,
                                                                 int n_ntiles, float* __restrict__ out) {
    pdl_prologue();
    __shared__ float acc[SC_NT * SC_PITCH];
    __shared__ int cnt[SC_WARPS][SC_CELLS];  // per-warp counts, then each warp's placement cursor per cell
    __shared__ int start[SC_CELLS + 1];      // the chunk's entities of cell c are list[start[c] .. start[c + 1])
    __shared__ int ecell[SC_CHUNK];
    __shared__ int list[SC_CHUNK];
    __shared__ int wsum[SC_WARPS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long bid = blockIdx.x;
    const int ct = (int)(bid % n_ctiles);
    bid /= n_ctiles;
    const int nt = (int)(bid % n_ntiles);
    const long long b = bid / n_ntiles;
    const long long c0 = (long long)ct * SC_CELLS;
    const int cells = (int)min((long long)SC_CELLS, ix.HW - c0);
    const int n0 = nt * SC_NT;
    const bool lane_ok = n0 + lane < N;
    const float* xb = x + b * x_sb + (long long)(n0 + lane) * x_sn;
    for (int i = tid; i < SC_NT * SC_PITCH; i += SC_THREADS) acc[i] = 0.f;

    for (int m0 = 0; m0 < M; m0 += SC_CHUNK) {
        const int len = min(SC_CHUNK, M - m0);
        int any = 0;
        for (int i = tid; i < SC_CHUNK; i += SC_THREADS) {
            int cell = -1;
            if (i < len) {
                const long long idx = flat_index(ix, b, m0 + i);
                if (idx >= c0 && idx < c0 + cells) cell = (int)(idx - c0);
            }
            ecell[i] = cell;
            any |= cell >= 0;
        }
        for (int i = tid; i < SC_WARPS * SC_CELLS; i += SC_THREADS) (&cnt[0][0])[i] = 0;
        if (!__syncthreads_or(any)) continue;  // no entity of this chunk falls in the tile

        // count: warp w, its segment in rounds of 32 entities; the highest lane of each group of equal cells adds the group
        for (int r = 0; r < SC_SEG; r += 32) {
            const int cell = ecell[warp * SC_SEG + r + lane];
            const unsigned peers = __match_any_sync(FULL, cell);
            if (cell >= 0 && lane == 31 - __clz(peers)) cnt[warp][cell] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();

        // start[c]: entities of the chunk in cells < c; cnt[w][c]: start[c] + entities of cell c in the segments of warps < w
        int tot = 0;
        if (tid < SC_CELLS)
            for (int w = 0; w < SC_WARPS; ++w) {
                const int v = cnt[w][tid];
                cnt[w][tid] = tot;
                tot += v;
            }
        int incl = tot;
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(FULL, incl, d);
            if (lane >= d) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (tid < SC_CELLS) {
            int base = 0;
            for (int w = 0; w < warp; ++w) base += wsum[w];
            const int s = base + incl - tot;
            start[tid] = s;
            for (int w = 0; w < SC_WARPS; ++w) cnt[w][tid] += s;
            if (tid == SC_CELLS - 1) start[SC_CELLS] = base + incl;
        }
        __syncthreads();

        // place: the same rounds again, so the entities of a cell keep ascending m
        for (int r = 0; r < SC_SEG; r += 32) {
            const int i = warp * SC_SEG + r + lane;
            const int cell = ecell[i];
            const unsigned peers = __match_any_sync(FULL, cell);
            if (cell >= 0) list[cnt[warp][cell] + __popc(peers & ((1u << lane) - 1u))] = m0 + i;
            __syncwarp();
            if (cell >= 0 && lane == 31 - __clz(peers)) cnt[warp][cell] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();

        // accumulate: one warp per cell, lane = n
        for (int c = warp; c < cells; c += SC_WARPS) {
            const int s = start[c], e = start[c + 1];
            if (s == e || !lane_ok) continue;
            float v;
            if (COVER) {
                v = xb[(long long)list[e - 1] * x_sm];
            } else {
                v = acc[lane * SC_PITCH + c];
                int j = s;
                for (; j + 4 <= e; j += 4) {
                    const float a0 = xb[(long long)list[j] * x_sm], a1 = xb[(long long)list[j + 1] * x_sm];
                    const float a2 = xb[(long long)list[j + 2] * x_sm], a3 = xb[(long long)list[j + 3] * x_sm];
                    v = fadd(fadd(fadd(fadd(v, a0), a1), a2), a3);
                }
                for (; j < e; ++j) v = fadd(v, xb[(long long)list[j] * x_sm]);
            }
            acc[lane * SC_PITCH + c] = v;
        }
        __syncthreads();
    }

    __syncthreads();  // the zero fill, when no chunk ran
    const int rows = min(SC_NT, N - n0);
    float* ob = out + (b * N + n0) * ix.HW + c0;
    for (int r = warp; r < rows; r += SC_WARPS)
        for (int c = lane; c < cells; c += 32) ob[(long long)r * ix.HW + c] = acc[r * SC_PITCH + c];
}

// dense backward: CTA (b, cell tile, feature tile) stages g[b, n-tile, cell tile] and writes the d x rows of the entities in
// that cell tile; the first cell tile also writes the zero rows of b's out-of-range entities.  Each row is written by one
// CTA, so the order entities are found in does not change a bit.
__global__ void __launch_bounds__(SC_THREADS) scatter_bwd_tile_kernel(const float* __restrict__ g, long long g_sb, long long g_sn,
                                                                      long long g_sc, ScatterIndex ix, int M, int N,
                                                                      int n_ctiles, int n_ntiles, float* __restrict__ dx) {
    pdl_prologue();
    __shared__ float tile[SC_NT * SC_PITCH];
    __shared__ int ent[SC_THREADS];
    __shared__ int ent_cell[SC_THREADS];
    __shared__ int n_ent;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long bid = blockIdx.x;
    const int ct = (int)(bid % n_ctiles);
    bid /= n_ctiles;
    const int nt = (int)(bid % n_ntiles);
    const long long b = bid / n_ntiles;
    const long long c0 = (long long)ct * SC_CELLS;
    const int cells = (int)min((long long)SC_CELLS, ix.HW - c0);
    const int n0 = nt * SC_NT;
    const int rows = min(SC_NT, N - n0);
    const float* gb = g + b * g_sb + (long long)n0 * g_sn + c0 * g_sc;
    for (int r = warp; r < rows; r += SC_WARPS)
        for (int c = lane; c < cells; c += 32) tile[r * SC_PITCH + c] = __ldg(gb + r * g_sn + c * g_sc);

    for (int m0 = 0; m0 < M; m0 += SC_THREADS) {
        if (tid == 0) n_ent = 0;
        __syncthreads();
        const int m = m0 + tid;
        if (m < M) {
            const long long idx = flat_index(ix, b, m);
            int cell = -2;
            if (idx >= c0 && idx < c0 + cells)
                cell = (int)(idx - c0);
            else if ((idx < 0 || idx >= ix.HW) && ct == 0)
                cell = -1;
            if (cell != -2) {
                const int k = atomicAdd(&n_ent, 1);
                ent[k] = m;
                ent_cell[k] = cell;
            }
        }
        __syncthreads();
        const int k_n = n_ent;
        for (int k = warp; k < k_n; k += SC_WARPS) {
            const int cell = ent_cell[k];
            if (lane < rows) dx[(b * M + ent[k]) * N + n0 + lane] = cell >= 0 ? tile[lane * SC_PITCH + cell] : 0.f;
        }
        __syncthreads();
    }
}

// sparse backward: one thread per d x value, n fastest (coalesced stores), gathering g[b, n, idx] directly
__global__ void __launch_bounds__(SC_THREADS) scatter_bwd_gather_kernel(const float* __restrict__ g, long long g_sb,
                                                                        long long g_sn, long long g_sc, ScatterIndex ix,
                                                                        long long M, long long N, long long total,
                                                                        float* __restrict__ dx) {
    pdl_prologue();
    const long long stride = (long long)gridDim.x * SC_THREADS;
    for (long long i = (long long)blockIdx.x * SC_THREADS + threadIdx.x; i < total; i += stride) {
        const long long bm = i / N, n = i - bm * N;
        const long long b = bm / M, m = bm - b * M;
        const long long idx = flat_index(ix, b, m);
        dx[i] = (idx >= 0 && idx < ix.HW) ? __ldg(g + b * g_sb + n * g_sn + idx * g_sc) : 0.f;
    }
}

// the tile grid (b, feature tile, cell tile), flattened with the cell tile fastest; false when it does not fit a launch
bool tile_grid(long long B, long long N, long long HW, int& n_ctiles, int& n_ntiles, long long& grid) {
    const long long ctiles = (HW + SC_CELLS - 1) / SC_CELLS, ntiles = (N + SC_NT - 1) / SC_NT;
    if (ctiles > 0x7fffffffLL || ntiles > 0x7fffffffLL) return false;
    grid = B * ntiles * ctiles;
    n_ctiles = (int)ctiles;
    n_ntiles = (int)ntiles;
    return grid <= 0x7fffffffLL;
}

bool index_args_ok(const long long* row, const long long* col, long long B, long long M, long long N, long long H,
                   long long W) {
    if (B < 0 || M < 0 || N < 0 || H < 0 || W < 0 || M > 0x7fffffffLL || N > 0x7fffffffLL) return false;
    if (H > 0 && W > 0x7fffffffffffffffLL / H) return false;
    return B * M == 0 || (row && col);
}
}  // namespace
}  // namespace b200rl

extern "C" int b200rl_scatter_fwd(const float* x, long long x_sb, long long x_sm, long long x_sn, const long long* row,
                                  long long row_sb, long long row_sm, const long long* col, long long col_sb,
                                  long long col_sm, long long B, long long M, long long N, long long H, long long W, int mode,
                                  float* out, void* stream) {
    using namespace b200rl;
    if ((mode != B200RL_SCATTER_ADD && mode != B200RL_SCATTER_COVER) || !index_args_ok(row, col, B, M, N, H, W))
        return B200RL_ERR_ARG;
    const long long HW = H * W;
    if (B * N * HW == 0) return B200RL_OK;
    if (!out || (M > 0 && !x)) return B200RL_ERR_ARG;
    int n_ctiles, n_ntiles;
    long long grid;
    if (!tile_grid(B, N, HW, n_ctiles, n_ntiles, grid)) return B200RL_ERR_ARG;
    const ScatterIndex ix{row, row_sb, row_sm, col, col_sb, col_sm, W, HW};
    const cudaStream_t st = (cudaStream_t)stream;
    if (mode == B200RL_SCATTER_COVER)
        return launch_k(scatter_fwd_kernel<true>, (int)grid, SC_THREADS, 0, st, x, x_sb, x_sm, x_sn, ix, (int)M, (int)N,
                        n_ctiles, n_ntiles, out);
    return launch_k(scatter_fwd_kernel<false>, (int)grid, SC_THREADS, 0, st, x, x_sb, x_sm, x_sn, ix, (int)M, (int)N,
                    n_ctiles, n_ntiles, out);
}

extern "C" int b200rl_scatter_bwd(const float* g, long long g_sb, long long g_sn, long long g_sc, const long long* row,
                                  long long row_sb, long long row_sm, const long long* col, long long col_sb,
                                  long long col_sm, long long B, long long M, long long N, long long H, long long W,
                                  float* grad_x, void* stream) {
    using namespace b200rl;
    if (!index_args_ok(row, col, B, M, N, H, W)) return B200RL_ERR_ARG;
    const long long HW = H * W, total = B * M * N;
    if (total == 0) return B200RL_OK;
    if (!grad_x || (HW > 0 && !g)) return B200RL_ERR_ARG;
    const ScatterIndex ix{row, row_sb, row_sm, col, col_sb, col_sm, W, HW};
    const cudaStream_t st = (cudaStream_t)stream;
    int n_ctiles, n_ntiles;
    long long grid;
    if (HW > 0 && M * SC_SECTOR_FLOATS >= HW && tile_grid(B, N, HW, n_ctiles, n_ntiles, grid))
        return launch_k(scatter_bwd_tile_kernel, (int)grid, SC_THREADS, 0, st, g, g_sb, g_sn, g_sc, ix, (int)M, (int)N,
                        n_ctiles, n_ntiles, grad_x);
    grid = (total + SC_THREADS - 1) / SC_THREADS;
    if (grid > (long long)NUM_SMS * 16) grid = (long long)NUM_SMS * 16;
    return launch_k(scatter_bwd_gather_kernel, (int)grid, SC_THREADS, 0, st, g, g_sb, g_sn, g_sc, ix, M, N, total, grad_x);
}
