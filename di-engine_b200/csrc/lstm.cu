// The layer-normalised LSTM step of ding/torch_utils/network/rnn.py:131-239 (lstm_type='normal', norm_type='LN'): all the
// work between the two GEMMs of a step.  The GEMMs themselves (x_t Wx, h_{t-1} Wh and their transposes in the backward)
// are the caller's.
//
// Step kernels: one CTA of LS_THREADS threads per batch row b.  Thread `tid` owns the hidden units j = tid + k*LS_THREADS,
// k < K, and for each of them the four gate columns g*H + j (g = i, f, o, u), so the gate split, the cell and the state
// stores need no exchange between threads; the two LayerNorm rows (4H each) are reduced across the CTA in a fixed order.
// K = ceil(H / LS_THREADS) in {1, 2, 4, 8} keeps both 4H rows in registers up to 4H = 4096; above that (K = 0) the same
// code re-reads the rows from global memory (L1 / L2 resident: one CTA reads its own 32 KB or more) in each pass.
// At B = 64, H = 512 the forward is 64 CTAs of 128 threads reading 2 x 8 KB each: a launch-latency-bound step.
//
// Parameter kernel: one CTA per 32 gate columns, LP_WARPS warps striding over all T*B rows (lane = column, coalesced);
// each lane sums in double, and the warps' sums are added in warp order, so the result does not depend on timing.
#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {
namespace {
constexpr int LS_THREADS = 128;
constexpr int LS_WARPS = LS_THREADS / 32;
constexpr int LS_MAX_K = 8;  // 4H <= 4 * LS_THREADS * LS_MAX_K = 4096 in registers
constexpr int LP_WARPS = 16;
constexpr float LN_EPS = 1e-5f;  // nn.LayerNorm's default, the only eps the Python side sends here

struct Row {  // a (rows, cols) operand: element (r, k) at p[r*sr + k*sk]
    const float* p;
    long long sr, sk;
    __device__ __forceinline__ float at(long long r, long long k) const { return p[r * sr + k * sk]; }
};
struct OutRow {
    float* p;
    long long sr, sk;
    __device__ __forceinline__ float& at(long long r, long long k) const { return p[r * sr + k * sk]; }
};
struct Vec {  // a (4H) parameter
    const float* p;
    long long s;
    __device__ __forceinline__ float at(long long k) const { return __ldg(p + k * s); }
};
struct LnParams {
    Vec gamma_x, beta_x, gamma_h, beta_h, bias;
};

// The pointwise math of a step (normalisation, gates, cell and their derivatives) runs in double and rounds once on the
// store: the step's rounding then stays well below the fp32 reference's, whose error grows with T, and the two GEMMs of a
// step stay the only fp32 arithmetic on the recurrence.
__device__ __forceinline__ double sigmoid_d(double v) { return 1.0 / (1.0 + exp(-v)); }

// sums of N per-thread values over the CTA, in double and a fixed order; every thread receives the totals.  The row
// statistics are shared by all 4H columns of the row, so their rounding does not average out downstream (d x = d_gx Wx^T
// sums 4H columns that carry the same error in mean(d x^)): double keeps them below the reference's error.
template <int N>
__device__ __forceinline__ void cta_sum(double (&v)[N], double (*red)[LS_WARPS]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int n = 0; n < N; ++n) {
        double r = v[n];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        if (lane == 0) red[n][warp] = r;
    }
    __syncthreads();
#pragma unroll
    for (int n = 0; n < N; ++n) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < LS_WARPS; ++w) s += red[n][w];
        v[n] = s;
    }
    __syncthreads();  // red is reused by the next call
}

// the two rows of one batch row: gx (x_t Wx) and gh (h_{t-1} Wh), before normalisation; in registers when K > 0
template <int K>
struct GateRows {
    static constexpr int KR = K > 0 ? K : 1;
    float ax[4][KR], ah[4][KR];
    Row gx, gh;
    long long b, H;
    int kn;

    __device__ __forceinline__ GateRows(const Row& gx_, const Row& gh_, long long b_, long long H_)
        : gx(gx_), gh(gh_), b(b_), H(H_), kn(K > 0 ? K : (int)((H_ + LS_THREADS - 1) / LS_THREADS)) {
        if constexpr (K > 0) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const long long j = threadIdx.x + (long long)k * LS_THREADS;
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    ax[g][k] = j < H ? gx.at(b, g * H + j) : 0.f;
                    ah[g][k] = j < H ? gh.at(b, g * H + j) : 0.f;
                }
            }
        }
    }
    __device__ __forceinline__ float x(int g, int k, long long j) const {
        if constexpr (K > 0) return ax[g][k];
        return gx.at(b, g * H + j);
    }
    __device__ __forceinline__ float h(int g, int k, long long j) const {
        if constexpr (K > 0) return ah[g][k];
        return gh.at(b, g * H + j);
    }

    // nn.LayerNorm's statistics of both rows: mean and 1/sqrt(biased variance + eps), the variance about the mean
    __device__ __forceinline__ void stats(double (*red)[LS_WARPS], double& mx, double& rx, double& mh, double& rh) const {
        double s[2] = {0.0, 0.0};
#pragma unroll
        for (int k = 0; k < (K > 0 ? K : kn); ++k) {
            const long long j = threadIdx.x + (long long)k * LS_THREADS;
            if (j < H)
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    s[0] += x(g, k, j);
                    s[1] += h(g, k, j);
                }
        }
        cta_sum<2>(s, red);
        const double n = (double)(4 * H);
        mx = s[0] / n;
        mh = s[1] / n;
        double q[2] = {0.0, 0.0};
#pragma unroll
        for (int k = 0; k < (K > 0 ? K : kn); ++k) {
            const long long j = threadIdx.x + (long long)k * LS_THREADS;
            if (j < H)
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const double dx = (double)x(g, k, j) - mx, dh = (double)h(g, k, j) - mh;
                    q[0] = fma(dx, dx, q[0]);
                    q[1] = fma(dh, dh, q[1]);
                }
        }
        cta_sum<2>(q, red);
        rx = 1.0 / sqrt(q[0] / n + (double)LN_EPS);
        rh = 1.0 / sqrt(q[1] / n + (double)LN_EPS);
    }
};

// the pre-activation of gate column gj: LN_x(gx) + LN_h(gh), then + bias (rnn.py:219-222)
__device__ __forceinline__ double gate_pre(const LnParams& p, long long gj, double xh, double hh) {
    const double lx = fma(xh, (double)p.gamma_x.at(gj), (double)p.beta_x.at(gj));
    const double lh = fma(hh, (double)p.gamma_h.at(gj), (double)p.beta_h.at(gj));
    return (lx + lh) + (double)p.bias.at(gj);
}

template <int K>
__global__ void __launch_bounds__(LS_THREADS) lnlstm_fwd_kernel(Row gx, Row gh, LnParams p, Row c_prev, long long H,
                                                                OutRow h_out, OutRow c_out, OutRow h_next, OutRow c_next,
                                                                float* __restrict__ stats, long long st_sr) {
    pdl_prologue();
    __shared__ double red[2][LS_WARPS];
    const long long b = blockIdx.x;
    const GateRows<K> rows(gx, gh, b, H);
    double mx, rx, mh, rh;
    rows.stats(red, mx, rx, mh, rh);
#pragma unroll
    for (int k = 0; k < (K > 0 ? K : rows.kn); ++k) {
        const long long j = threadIdx.x + (long long)k * LS_THREADS;
        if (j >= H) continue;
        double a[4];
#pragma unroll
        for (int g = 0; g < 4; ++g)
            a[g] = gate_pre(p, g * H + j, (rows.x(g, k, j) - mx) * rx, (rows.h(g, k, j) - mh) * rh);
        const double i = sigmoid_d(a[0]), f = sigmoid_d(a[1]), o = sigmoid_d(a[2]), u = tanh(a[3]);
        const float c = (float)(f * c_prev.at(b, j) + i * u);
        const float h = (float)(o * tanh((double)c));
        h_out.at(b, j) = h;
        c_out.at(b, j) = c;
        if (h_next.p) h_next.at(b, j) = h;
        if (c_next.p) c_next.at(b, j) = c;
    }
    if (stats && threadIdx.x == 0) {
        float* s = stats + b * st_sr;
        s[0] = (float)mx;
        s[1] = (float)rx;
        s[2] = (float)mh;
        s[3] = (float)rh;
    }
}

struct BwdIn {
    Row dy, dh_rec, dc_in;  // each nullable (p == nullptr reads as zero)
    const float* stats;
    long long st_sr;
    Row c_prev, c;
};
struct BwdOut {
    OutRow d_gx, d_gh, d_gate, dc_prev;
};

__device__ __forceinline__ float ld_or0(const Row& r, long long b, long long j) { return r.p ? r.at(b, j) : 0.f; }

template <int K>
__global__ void __launch_bounds__(LS_THREADS) lnlstm_bwd_kernel(Row gx, Row gh, LnParams p, BwdIn in, long long H,
                                                                BwdOut out) {
    pdl_prologue();
    __shared__ double red[4][LS_WARPS];
    constexpr bool KEEP_DG = K > 0 && K <= 4;  // at K = 8 the gate gradients would spill: re-read the own stores instead
    constexpr int KR = KEEP_DG ? K : 1;
    const long long b = blockIdx.x;
    const GateRows<K> rows(gx, gh, b, H);
    const float* st = in.stats + b * in.st_sr;
    const double mx = st[0], rx = st[1], mh = st[2], rh = st[3];
    float dg[4][KR];
    double s[4] = {0.0, 0.0, 0.0, 0.0};  // sum dx^, sum dx^ * x^, sum dh^, sum dh^ * h^
#pragma unroll
    for (int k = 0; k < (K > 0 ? K : rows.kn); ++k) {
        const long long j = threadIdx.x + (long long)k * LS_THREADS;
        if (j >= H) continue;
        double a[4], xh[4], hh[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            xh[g] = (rows.x(g, k, j) - mx) * rx;
            hh[g] = (rows.h(g, k, j) - mh) * rh;
            a[g] = gate_pre(p, g * H + j, xh[g], hh[g]);
        }
        const double i = sigmoid_d(a[0]), f = sigmoid_d(a[1]), o = sigmoid_d(a[2]), u = tanh(a[3]);
        const double tc = tanh((double)in.c.at(b, j));
        const double dh = (double)ld_or0(in.dy, b, j) + (double)ld_or0(in.dh_rec, b, j);
        const double dc = (double)ld_or0(in.dc_in, b, j) + dh * o * (1.0 - tc * tc);
        out.dc_prev.at(b, j) = (float)(dc * f);  // after the read of dc_in: dc_prev may be dc_in
        float d[4];
        d[0] = (float)(dc * u * i * (1.0 - i));
        d[1] = (float)(dc * in.c_prev.at(b, j) * f * (1.0 - f));
        d[2] = (float)(dh * tc * o * (1.0 - o));
        d[3] = (float)(dc * i * (1.0 - u * u));
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            out.d_gate.at(b, g * H + j) = d[g];
            if constexpr (KEEP_DG) dg[g][k] = d[g];
            const double dxh = (double)d[g] * p.gamma_x.at(g * H + j), dhh = (double)d[g] * p.gamma_h.at(g * H + j);
            s[0] += dxh;
            s[1] = fma(dxh, xh[g], s[1]);
            s[2] += dhh;
            s[3] = fma(dhh, hh[g], s[3]);
        }
    }
    cta_sum<4>(s, red);
    const double n = (double)(4 * H);
    const double mdx = s[0] / n, mdxx = s[1] / n, mdh = s[2] / n, mdhh = s[3] / n;
#pragma unroll
    for (int k = 0; k < (K > 0 ? K : rows.kn); ++k) {
        const long long j = threadIdx.x + (long long)k * LS_THREADS;
        if (j >= H) continue;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const long long gj = g * H + j;
            float d;
            if constexpr (KEEP_DG) d = dg[g][k];
            else d = out.d_gate.at(b, gj);  // this thread's own store above
            const double xh = (rows.x(g, k, j) - mx) * rx, hh = (rows.h(g, k, j) - mh) * rh;
            out.d_gx.at(b, gj) = (float)(rx * ((double)d * p.gamma_x.at(gj) - mdx - xh * mdxx));
            out.d_gh.at(b, gj) = (float)(rh * ((double)d * p.gamma_h.at(gj) - mdh - hh * mdhh));
        }
    }
}

__global__ void __launch_bounds__(LP_WARPS * 32) lnlstm_param_kernel(Row d_gate, Row gx, Row gh, const float* __restrict__ stats,
                                                                    long long st_sr, long long R, long long G,
                                                                    OutRow d_gamma_x, OutRow d_gamma_h, OutRow d_beta) {
    pdl_prologue();
    __shared__ double red[3][LP_WARPS][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long col = (long long)blockIdx.x * 32 + lane;
    double sx = 0.0, sh = 0.0, sb = 0.0;
    if (col < G)
        for (long long r = warp; r < R; r += LP_WARPS) {
            const float* st = stats + r * st_sr;
            const float d = d_gate.at(r, col);
            const float xh = (gx.at(r, col) - __ldg(st)) * __ldg(st + 1);
            const float hh = (gh.at(r, col) - __ldg(st + 2)) * __ldg(st + 3);
            sx += (double)(d * xh);
            sh += (double)(d * hh);
            sb += (double)d;
        }
    red[0][warp][lane] = sx;
    red[1][warp][lane] = sh;
    red[2][warp][lane] = sb;
    __syncthreads();
    if (warp == 0 && col < G) {
        double t[3] = {0.0, 0.0, 0.0};
        for (int w = 0; w < LP_WARPS; ++w)
#pragma unroll
            for (int q = 0; q < 3; ++q) t[q] += red[q][w][lane];
        d_gamma_x.at(0, col) = (float)t[0];
        d_gamma_h.at(0, col) = (float)t[1];
        d_beta.at(0, col) = (float)t[2];
    }
}

// K for a hidden size: the register path's units per thread, or 0 for the re-reading path
int units_per_thread(long long H) {
    const long long k = (H + LS_THREADS - 1) / LS_THREADS;
    if (k <= 1) return 1;
    if (k <= 2) return 2;
    if (k <= 4) return 4;
    if (k <= LS_MAX_K) return LS_MAX_K;
    return 0;
}

bool sizes_ok(long long B, long long H) { return B >= 0 && B <= 0x7fffffffLL && H >= 1 && H <= (1LL << 40); }
}  // namespace
}  // namespace b200rl

extern "C" int b200rl_lnlstm_step_fwd(const float* gx, long long gx_sb, long long gx_sk, const float* gh, long long gh_sb,
                                      long long gh_sk, const float* gamma_x, long long gamma_x_s, const float* beta_x,
                                      long long beta_x_s, const float* gamma_h, long long gamma_h_s, const float* beta_h,
                                      long long beta_h_s, const float* bias, long long bias_s, const float* c_prev,
                                      long long cp_sb, long long cp_sk, long long B, long long H, float* h, long long h_sb,
                                      long long h_sk, float* c, long long c_sb, long long c_sk, float* h_next,
                                      long long hn_sb, long long hn_sk, float* c_next, long long cn_sb, long long cn_sk,
                                      float* stats, long long st_sb, void* stream) {
    using namespace b200rl;
    if (!sizes_ok(B, H)) return B200RL_ERR_ARG;
    if (B == 0) return B200RL_OK;
    if (!gx || !gh || !gamma_x || !beta_x || !gamma_h || !beta_h || !bias || !c_prev || !h || !c) return B200RL_ERR_ARG;
    const Row rgx{gx, gx_sb, gx_sk}, rgh{gh, gh_sb, gh_sk}, rcp{c_prev, cp_sb, cp_sk};
    const LnParams p{{gamma_x, gamma_x_s}, {beta_x, beta_x_s}, {gamma_h, gamma_h_s}, {beta_h, beta_h_s}, {bias, bias_s}};
    const OutRow ho{h, h_sb, h_sk}, co{c, c_sb, c_sk}, hn{h_next, hn_sb, hn_sk}, cn{c_next, cn_sb, cn_sk};
    const cudaStream_t st = (cudaStream_t)stream;
#define B200RL_LNLSTM_FWD(K) \
    launch_k(lnlstm_fwd_kernel<K>, (int)B, LS_THREADS, 0, st, rgx, rgh, p, rcp, H, ho, co, hn, cn, stats, st_sb)
    switch (units_per_thread(H)) {
        case 1: return B200RL_LNLSTM_FWD(1);
        case 2: return B200RL_LNLSTM_FWD(2);
        case 4: return B200RL_LNLSTM_FWD(4);
        case 8: return B200RL_LNLSTM_FWD(8);
        default: return B200RL_LNLSTM_FWD(0);
    }
#undef B200RL_LNLSTM_FWD
}

extern "C" int b200rl_lnlstm_step_bwd(const float* dy, long long dy_sb, long long dy_sk, const float* dh_rec,
                                      long long dhr_sb, long long dhr_sk, const float* dc_in, long long dci_sb,
                                      long long dci_sk, const float* gx, long long gx_sb, long long gx_sk, const float* gh,
                                      long long gh_sb, long long gh_sk, const float* stats, long long st_sb,
                                      const float* gamma_x, long long gamma_x_s, const float* beta_x, long long beta_x_s,
                                      const float* gamma_h, long long gamma_h_s, const float* beta_h, long long beta_h_s,
                                      const float* bias, long long bias_s, const float* c_prev, long long cp_sb,
                                      long long cp_sk, const float* c, long long c_sb, long long c_sk, long long B,
                                      long long H, float* d_gx, long long dgx_sb, long long dgx_sk, float* d_gh,
                                      long long dgh_sb, long long dgh_sk, float* d_gate, long long dg_sb, long long dg_sk,
                                      float* dc_prev, long long dcp_sb, long long dcp_sk, void* stream) {
    using namespace b200rl;
    if (!sizes_ok(B, H)) return B200RL_ERR_ARG;
    if (B == 0) return B200RL_OK;
    if (!gx || !gh || !stats || !gamma_x || !beta_x || !gamma_h || !beta_h || !bias || !c_prev || !c || !d_gx || !d_gh ||
        !d_gate || !dc_prev)
        return B200RL_ERR_ARG;
    const Row rgx{gx, gx_sb, gx_sk}, rgh{gh, gh_sb, gh_sk};
    const LnParams p{{gamma_x, gamma_x_s}, {beta_x, beta_x_s}, {gamma_h, gamma_h_s}, {beta_h, beta_h_s}, {bias, bias_s}};
    const BwdIn in{{dy, dy_sb, dy_sk}, {dh_rec, dhr_sb, dhr_sk}, {dc_in, dci_sb, dci_sk}, stats, st_sb,
                   {c_prev, cp_sb, cp_sk}, {c, c_sb, c_sk}};
    const BwdOut out{{d_gx, dgx_sb, dgx_sk}, {d_gh, dgh_sb, dgh_sk}, {d_gate, dg_sb, dg_sk}, {dc_prev, dcp_sb, dcp_sk}};
    const cudaStream_t st = (cudaStream_t)stream;
#define B200RL_LNLSTM_BWD(K) launch_k(lnlstm_bwd_kernel<K>, (int)B, LS_THREADS, 0, st, rgx, rgh, p, in, H, out)
    switch (units_per_thread(H)) {
        case 1: return B200RL_LNLSTM_BWD(1);
        case 2: return B200RL_LNLSTM_BWD(2);
        case 4: return B200RL_LNLSTM_BWD(4);
        case 8: return B200RL_LNLSTM_BWD(8);
        default: return B200RL_LNLSTM_BWD(0);
    }
#undef B200RL_LNLSTM_BWD
}

extern "C" int b200rl_lnlstm_param_grads(const float* d_gate, long long dg_sr, long long dg_sk, const float* gx,
                                         long long gx_sr, long long gx_sk, const float* gh, long long gh_sr,
                                         long long gh_sk, const float* stats, long long st_sr, long long R, long long H,
                                         float* d_gamma_x, long long dgx_s, float* d_gamma_h, long long dgh_s,
                                         float* d_beta, long long db_s, void* stream) {
    using namespace b200rl;
    if (R < 0 || H < 1 || 4 * H / 32 >= 0x7fffffffLL) return B200RL_ERR_ARG;
    if (!d_gamma_x || !d_gamma_h || !d_beta || (R > 0 && (!d_gate || !gx || !gh || !stats))) return B200RL_ERR_ARG;
    const long long G = 4 * H;
    return launch_k(lnlstm_param_kernel, (int)((G + 31) / 32), LP_WARPS * 32, 0, (cudaStream_t)stream,
                    Row{d_gate, dg_sr, dg_sk}, Row{gx, gx_sr, gx_sk}, Row{gh, gh_sr, gh_sk}, stats, st_sr, R, G,
                    OutRow{d_gamma_x, 0, dgx_s}, OutRow{d_gamma_h, 0, dgh_s}, OutRow{d_beta, 0, db_s});
}
