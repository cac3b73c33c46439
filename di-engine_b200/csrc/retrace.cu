// compute_q_retraces (ding/rl_utils/retrace.py:7-56): ACER's Retrace(lambda) targets, a reverse scan along T with two gathers
// per step.  No gradient (the reference computes it under torch.no_grad(), policy/acer.py:231-232).
//
//   Qret[T] = V[T];  tmp = V[T]
//   for t = T-1 .. 0:   Qret[t] = r[t] + (gamma * w[t]) * tmp
//                       tmp     = min(ratio[t, a_t], 1) * (Qret[t] - Q[t, a_t]) + V[t]
//
// A CTA owns 32 batch columns.  Time is walked newest-first in chunks of 64 steps: ALL 256 threads gather the chunk's operands
// (action -> Q[t, a], ratio[t, a]; two dependent loads, 8 independent elements per thread) into shared memory, then one warp
// (lane = column) runs the dependent chain on them and the finished rows are stored coalesced.  A first version with one thread
// per column doing its own gathers pays T x 2 dependent DRAM latencies in a row.
// Separate round-to-nearest multiplies and adds in the reference's order: bit-identical.
// Algorithmic traffic: 28 B + one sector each of the two gathered rows per transition.
#include "../../include/b200rl.h"
#include "common.cuh"

namespace b200rl {

constexpr int RT_TC = 32;   // columns per CTA
constexpr int RT_CH = 64;   // time steps per chunk
constexpr int RT_NT = 256;

__global__ void __launch_bounds__(RT_NT) retrace_kernel(const float* __restrict__ q, const float* __restrict__ v,
                                                        const float* __restrict__ reward, const long long* __restrict__ action,
                                                        const float* __restrict__ weight, const float* __restrict__ ratio,
                                                        long long T, long long B, long long N, float gamma,
                                                        float* __restrict__ out) {
    pdl_prologue();
    __shared__ float s_r[RT_CH][RT_TC], s_gw[RT_CH][RT_TC], s_c[RT_CH][RT_TC], s_qa[RT_CH][RT_TC], s_v[RT_CH][RT_TC];
    const int tid = threadIdx.x;
    const long long c0 = (long long)blockIdx.x * RT_TC;
    const int W = (int)((B - c0) < RT_TC ? (B - c0) : RT_TC);
    float tmp = 0.f;
    if (tid < W) {
        tmp = v[T * B + c0 + tid];
        out[T * B + c0 + tid] = tmp;
    }
    for (long long hi = T; hi > 0; hi -= RT_CH) {
        const long long lo = hi > RT_CH ? hi - RT_CH : 0;
        const int rows = (int)(hi - lo);
        // ---- gather: element i -> (row j = i / 32 counted from the chunk's oldest step, column i % 32)
        for (int i = tid; i < rows * RT_TC; i += RT_NT) {
            const int j = i / RT_TC, c = i % RT_TC;
            if (c < W) {
                const long long e = (lo + j) * B + c0 + c;
                const long long a = action[e];
                s_r[j][c] = reward[e];
                s_gw[j][c] = fmul(gamma, weight[e]);
                s_v[j][c] = v[e];
                const float ra = ratio[e * N + a];
                s_c[j][c] = ra != ra ? ra : fminf(ra, 1.0f);  // clamp(max=1) keeps NaN
                s_qa[j][c] = q[e * N + a];
            }
        }
        __syncthreads();
        // ---- scan: lane = column, newest row first; Qret overwrites the reward slot
        if (tid < W) {
            for (int j = rows - 1; j >= 0; --j) {
                const float qr = fadd(s_r[j][tid], fmul(s_gw[j][tid], tmp));
                s_r[j][tid] = qr;
                tmp = fadd(fmul(s_c[j][tid], fsub(qr, s_qa[j][tid])), s_v[j][tid]);
            }
        }
        __syncthreads();
        for (int i = tid; i < rows * RT_TC; i += RT_NT) {
            const int j = i / RT_TC, c = i % RT_TC;
            if (c < W) out[(lo + j) * B + c0 + c] = s_r[j][c];
        }
        __syncthreads();
    }
}

}  // namespace b200rl

extern "C" int b200rl_q_retraces(const float* q_values, const float* v_pred, const float* rewards, const long long* actions,
                                 const float* weights, const float* ratio, long long T, long long B, long long N,
                                 double gamma, float* q_retraces, void* stream) {
    using namespace b200rl;
    if (T < 0 || B < 1 || N < 1 || !v_pred || !q_retraces) return B200RL_ERR_ARG;
    if (T > 0 && (!q_values || !rewards || !actions || !weights || !ratio)) return B200RL_ERR_ARG;
    return launch_k(retrace_kernel, div_up(B, RT_TC), RT_NT, 0, (cudaStream_t)stream, q_values, v_pred, rewards, actions, weights,
                    ratio, T, B, N, (float)gamma, q_retraces);
}
