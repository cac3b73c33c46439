// GAE reverse scan -- replaces the Python `for t in reversed(range(T))` of ding/rl_utils/gae.py:65-69.
//
// Layout: value/next_value/adv are (T, C) row-major with C = B (or B*A for the multi-agent case, gae.py:56-59);
// reward/done/traj_flag are (T, C/A) and broadcast over the trailing A.
//
// One CTA owns TC consecutive columns for all T (see gae_ws_kernel):
//   loader warps (fully parallel, float4 coalesced): nv' = nv*(1-done) (written back only where it changed -- the
//            reference mutates the caller's tensor, gae.py:61), delta = (r + g*nv') - v, f = gl*(1-traj) -> shared memory
//   scan warp (lane = column): A_t = delta_t + f_t*A_{t+1}; separate round-to-nearest mul and add in the reference's
//            order, so the result is bit-identical to the torch loop; adv is stored straight from the scan registers.
// T is processed in 128-row slabs from the end of the trajectory, each slab in four 32-row chunks handed from the
// loaders to the scan warp through named barriers; the carry stays in the scan lanes' registers.
// Algorithmic traffic: 5 reads + 1 write = 24 B per transition.
#include "../../include/b200rl.h"
#include "gae_tile.cuh"

namespace b200rl {

// Warp-specialised tile kernel.  A CTA owns TC columns; warp 0 is the scan warp, the other TC/4 warps are loaders.
// Loaders issue every 16-byte load of a 128-row slab up front (20 in flight per thread), newest rows first, then turn
// each 32-row chunk into (delta, f) pairs in shared memory and signal the chunk's named barrier.  The scan warp walks
// the chunks as they arrive -- the sequential part of chunk k overlaps the HBM latency of chunks k+1.. -- and stores
// adv straight from registers.  (Body: gae_tile.cuh.)
template <int TC, bool VEC>
__global__ void __launch_bounds__((TC / 4 + 1) * 32) gae_ws_kernel(
    const float* __restrict__ value, float* __restrict__ next_value, const float* __restrict__ reward,
    const float* __restrict__ done, const float* __restrict__ traj, float* __restrict__ adv, long long T,
    long long C, long long A, float gamma, float gl, int mask_inplace, float vscale) {
    pdl_prologue();
    __shared__ __align__(16) float s_d[GAE_NCHUNK][GAE_CH][TC];
    __shared__ __align__(16) float s_f[GAE_NCHUNK][GAE_CH][TC];
    gae_tile_body<TC, VEC>(value, next_value, reward, done, traj, adv, T, C, A, gamma, gl, mask_inplace,
                           (long long)blockIdx.x * TC, s_d, s_f, [](long long, bool) {}, vscale);
}

template <int TC>
static int launch_gae(const float* value, float* next_value, const float* reward, const float* done,
                      const float* traj, float* adv, long long T, long long C, long long A, float gamma, float gl,
                      int mask_inplace, bool vec, cudaStream_t st, float vscale) {
    const int grid = div_up(C, TC);
    constexpr int NT = (TC / 4 + 1) * 32;
    if (vec)
        return launch_k(gae_ws_kernel<TC, true>, grid, NT, 0, st, value, next_value, reward, done, traj, adv, T, C, A, gamma,
                        gl, mask_inplace, vscale);
    return launch_k(gae_ws_kernel<TC, false>, grid, NT, 0, st, value, next_value, reward, done, traj, adv, T, C, A, gamma,
                    gl, mask_inplace, vscale);
}

}  // namespace b200rl

namespace b200rl {
int gae_scan(const float* value, float* next_value, const float* reward, const float* done, const float* traj_flag, float* adv,
             long long T, long long C, long long A, double gamma_d, double lambda_d, int mask_next_value_inplace,
             float vscale, void* stream);
}

extern "C" int b200rl_gae(const float* value, float* next_value, const float* reward, const float* done,
                          const float* traj_flag, float* adv, long long T, long long C, long long A, double gamma_d,
                          double lambda_d, int mask_next_value_inplace, void* stream) {
    return b200rl::gae_scan(value, next_value, reward, done, traj_flag, adv, T, C, A, gamma_d, lambda_d,
                            mask_next_value_inplace, 0.f, stream);
}

// vscale != 0: value and next_value are multiplied by it on load (PPOPolicy's value_norm, ding/policy/ppo.py:276-278)
int b200rl::gae_scan(const float* value, float* next_value, const float* reward, const float* done, const float* traj_flag,
                     float* adv, long long T, long long C, long long A, double gamma_d, double lambda_d,
                     int mask_next_value_inplace, float vscale, void* stream) {
    using namespace b200rl;
    // python scalars reach torch as fp32(gamma) and fp32(gamma*lambda_) (product taken in double), gae.py:62-63
    const float gamma = (float)gamma_d, gamma_lambda = (float)(gamma_d * lambda_d);
    if (T < 0 || C < 0 || A < 1 || (C % A) != 0) return B200RL_ERR_ARG;
    if (T == 0 || C == 0) return B200RL_OK;
    if (!value || !next_value || !reward || !adv) return B200RL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    bool vec = (A == 1) && (C % 4 == 0) && aligned16(value) && aligned16(next_value) && aligned16(reward) &&
               aligned16(adv) && (!done || aligned16(done)) && (!traj_flag || aligned16(traj_flag));
    // column-tile width: the widest tile that still gives every SM at least ~2 CTAs
    if (C >= 32 * 2 * NUM_SMS)
        return launch_gae<32>(value, next_value, reward, done, traj_flag, adv, T, C, A, gamma, gamma_lambda,
                              mask_next_value_inplace, vec, st, vscale);
    if (C >= 16 * 2 * NUM_SMS)
        return launch_gae<16>(value, next_value, reward, done, traj_flag, adv, T, C, A, gamma, gamma_lambda,
                              mask_next_value_inplace, vec, st, vscale);
    return launch_gae<8>(value, next_value, reward, done, traj_flag, adv, T, C, A, gamma, gamma_lambda,
                         mask_next_value_inplace, vec, st, vscale);
}
