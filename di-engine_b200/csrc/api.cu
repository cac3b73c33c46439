// Library-level entry points of the C ABI declared in include/b200rl.h.
#include "../../include/b200rl.h"
#include "common.cuh"

#include <mutex>

// ---------------------------------------------------------------------------------------------------------------
// The record of the step chain on each (device, stream) (common.cuh): the capture it belongs to, the node of its last
// launch, and the bytes its launches may write since the last column kernel.
// ---------------------------------------------------------------------------------------------------------------
namespace b200rl {
namespace {
constexpr int CHAIN_STREAMS = 8;  // streams per device with a record; the oldest record gives way
constexpr int CHAIN_SPANS = 16;   // write spans per record (a column kernel + finalize + check report 11 at most)
struct StepChain {
    cudaStream_t st;
    unsigned long long id;
    void* last;  // null: no record
    int n;
    ByteSpan w[CHAIN_SPANS];
};
StepChain g_chain[MAX_DEVICES][CHAIN_STREAMS];
int g_chain_next[MAX_DEVICES];
std::mutex g_chain_mu;

StepChain* chain_of(int dev, cudaStream_t st) {
    for (StepChain& c : g_chain[dev])
        if (c.last && c.st == st) return &c;
    return nullptr;
}
bool overlaps(const ByteSpan& a, const ByteSpan& b) { return a.lo < b.hi && b.lo < a.hi; }
}  // namespace

ChainPoint capture_now(cudaStream_t st) {
    ChainPoint at{};
    if (current_device(at.dev) != B200RL_OK) return at;
    cudaStreamCaptureStatus s;
    const cudaGraphNode_t* deps = nullptr;
    size_t nd = 0;
    // a stream that cannot be queried is treated as not captured: the launch itself reports what is wrong with it
    if (cuda_rc(cudaStreamGetCaptureInfo(st, &s, &at.id, nullptr, &deps, &nd)) != B200RL_OK) return at;
    at.capturing = s == cudaStreamCaptureStatusActive;
    at.dep = (at.capturing && nd == 1) ? (void*)deps[0] : nullptr;
    return at;
}

bool chain_may_defer(cudaStream_t st, const ChainPoint& at, const ByteSpan* reads, int n_reads) {
    if (!at.capturing || !at.dep || !pdl_enabled()) return false;
    std::lock_guard<std::mutex> lock(g_chain_mu);
    const StepChain* c = chain_of(at.dev, st);
    if (!c || c->id != at.id || c->last != at.dep) return false;
    for (int i = 0; i < n_reads; ++i)
        for (int k = 0; k < c->n; ++k)
            if (overlaps(reads[i], c->w[k])) return false;
    return true;
}

void chain_report(cudaStream_t st, const ChainPoint& at, bool starts, const ByteSpan* writes, int n_writes) {
    std::lock_guard<std::mutex> lock(g_chain_mu);
    StepChain* c = chain_of(at.dev, st);
    ChainPoint now{};
    if (at.capturing) now = capture_now(st);
    // the chain goes on only where this launch followed it directly (a check) or starts it, in the same capture
    const bool follows = c && c->id == at.id && at.dep && c->last == at.dep;
    if (!now.capturing || !now.dep || now.id != at.id || (!starts && !follows) ||
        (starts ? 0 : c->n) + n_writes > CHAIN_SPANS) {
        if (c) c->last = nullptr;
        return;
    }
    if (!c) {
        c = &g_chain[at.dev][g_chain_next[at.dev]];
        g_chain_next[at.dev] = (g_chain_next[at.dev] + 1) % CHAIN_STREAMS;
    }
    if (starts) c->n = 0;
    c->st = st;
    c->id = at.id;
    c->last = now.dep;
    for (int i = 0; i < n_writes; ++i) c->w[c->n++] = writes[i];
}
}  // namespace b200rl

extern "C" int b200rl_version(void) { return 115; }
extern "C" int b200rl_built_for_sm(void) { return 90; }
extern "C" size_t b200rl_workspace_bytes(void) { return (size_t)WS_MIN_BYTES; }

// ---------------------------------------------------------------------------------------------------------------
// Bandwidth probe (tools/calib_copy.py): a plain persistent float4 copy with 8 independent 16-byte loads in flight per
// thread.  It calibrates what a well-formed streaming kernel reaches at the (small) byte counts of this path, where
// launch ramp-up and DRAM latency are a large share of the run time and the 2 GiB-copy peak is out of reach.
// ---------------------------------------------------------------------------------------------------------------
namespace b200rl {
__global__ void __launch_bounds__(256) probe_copy_kernel(const float4* __restrict__ src, float4* __restrict__ dst,
                                                         long long n) {
    pdl_prologue();
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 7 * stride < n; i += 8 * stride) {
        float4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = __ldcs(src + i + k * stride);
#pragma unroll
        for (int k = 0; k < 8; ++k) __stcs(dst + i + k * stride, v[k]);
    }
    for (; i < n; i += stride) __stcs(dst + i, __ldcs(src + i));
}
}  // namespace b200rl

extern "C" int b200rl_probe_copy(const float* src, float* dst, long long n_floats, int ctas_per_sm, void* stream) {
    if (!src || !dst || n_floats < 0 || (n_floats & 3) || ctas_per_sm < 1) return B200RL_ERR_ARG;
    const long long n4 = n_floats / 4;
    long long grid = (long long)b200rl::NUM_SMS * ctas_per_sm;
    const long long need = (n4 + 255) / 256;
    if (grid > need) grid = need > 0 ? need : 1;
    return b200rl::launch_k(b200rl::probe_copy_kernel, (int)grid, 256, 0, (cudaStream_t)stream, reinterpret_cast<const float4*>(src),
                                                                           reinterpret_cast<float4*>(dst), n4);
}

// ---------------------------------------------------------------------------------------------------------------
// One-shot all-reduce (mean) of up to 8 floats over NVLink peer memory -- the only exchange step of this path in data
// parallel training (the packed loss scalars; SURVEY section 8e).  Every rank owns a mailbox in symmetric (peer-mapped)
// memory, [2 slots][world][8 floats + sequence word]; the kernel is ONE small CTA:
//   - lane (r, j) stores this rank's value j into peer r's mailbox (plain stores over NVLink), then publishes the step's
//     sequence number there with a system-scope release store;
//   - lane r waits until peer r's sequence number has arrived in the local mailbox (acquire loads), then lanes j add the
//     world values in rank order -- identical, deterministic result on every rank -- and divide by the world size
//     (the reference's all_reduce + div_(world_size), ding/utils/pytorch_ddp_dist_helper.py:38-47).
// Latency is one NVLink store + flag round (~ a few us) instead of a small-message NCCL all-reduce, nothing else runs on
// the SMs for it, and being an ordinary kernel it can be captured in the step's CUDA graph.  Two mailbox slots alternate by
// sequence parity: a rank cannot be two steps ahead of a peer because it needs that peer's flag to finish a step.
// ---------------------------------------------------------------------------------------------------------------
namespace b200rl {
constexpr int P2P_VALS = 8;
constexpr int P2P_ENTRY = 16;  // floats per (slot, rank) entry: 8 values, 1 sequence word, padding to 64 bytes

__global__ void __launch_bounds__(256) p2p_allreduce_mean_kernel(const float* __restrict__ local,
                                                                 const unsigned long long* __restrict__ mailboxes,
                                                                 int rank, int world, int n, unsigned int* seq_dev,
                                                                 float* __restrict__ out) {
    pdl_prologue();
    __shared__ float s_val[64][P2P_VALS];
    const unsigned int seq = *seq_dev + 1u;  // sequence number of this exchange (same on every rank)
    const int slot = (int)(seq & 1u);
    const int tid = threadIdx.x;
    // ---- scatter: thread (r, j), r = tid / 8 (peer), j = tid % 8 (value); warp-uniform trip count ----
    for (int r0 = 0; r0 < world; r0 += 256 / P2P_VALS) {
        const int r = r0 + tid / P2P_VALS, j = tid % P2P_VALS;
        const bool act = r < world;
        float* peer = act ? reinterpret_cast<float*>(mailboxes[r]) + ((size_t)slot * world + rank) * P2P_ENTRY : nullptr;
        if (act && j < n) peer[j] = local[j];
        __threadfence_system();  // this lane's value is visible system-wide ...
        __syncwarp();
        if (act && j == 0)       // ... before the sequence word that announces the entry
            asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(reinterpret_cast<unsigned int*>(peer + P2P_VALS)),
                         "r"(seq)
                         : "memory");
    }
    // ---- gather: thread r waits for peer r's flag in the LOCAL mailbox ----
    const float* mine = reinterpret_cast<const float*>(mailboxes[rank]) + (size_t)slot * world * P2P_ENTRY;
    for (int r = tid; r < world; r += 256) {
        const unsigned int* flag = reinterpret_cast<const unsigned int*>(mine + (size_t)r * P2P_ENTRY + P2P_VALS);
        unsigned int v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
            if (v != seq) __nanosleep(64);
        } while (v != seq);
        for (int j = 0; j < n; ++j) s_val[r & 63][j] = __ldcv(mine + (size_t)r * P2P_ENTRY + j);
    }
    __syncthreads();
    if (tid < n) {
        float acc = 0.f;
        for (int r = 0; r < world; ++r) acc += s_val[r][tid];
        out[tid] = acc / (float)world;
    }
    if (tid == 0) *seq_dev = seq;
}
}  // namespace b200rl

extern "C" int b200rl_p2p_allreduce_mean(const float* local, const unsigned long long* mailbox_ptrs_dev, int rank,
                                         int world, int n, unsigned int* seq_dev, float* out, void* stream) {
    if (!local || !mailbox_ptrs_dev || !seq_dev || !out || n < 1 || n > b200rl::P2P_VALS || world < 1 || world > 64 ||
        rank < 0 || rank >= world)
        return B200RL_ERR_ARG;
    return b200rl::launch_k(b200rl::p2p_allreduce_mean_kernel, 1, 256, 0, (cudaStream_t)stream, local, mailbox_ptrs_dev,
                            rank, world, n, seq_dev, out);
}

extern "C" size_t b200rl_p2p_mailbox_floats(int world) { return (size_t)2 * world * b200rl::P2P_ENTRY; }

// ---------------------------------------------------------------------------------------------------------------
// Tail of the exchange that rides on the learner step's own launches (common.cuh): after the last step Q its values are
// staged but not published and tag Q-1 is published but not consumed (no next step): warp k of this small kernel consumes
// Q-1, publishes Q and consumes Q, so that out_mean[k] = mean over ranks of the LAST step's out[k] (out_mean[8+k]: step Q-1).
// Mailbox layout: [2 slots][world][8] 64-bit words {tag, value}; b200rl_p2p_mailbox_floats(world) floats hold exactly that.
// The tail is idempotent for the pipeline: the next step's kernel re-publishes tag Q (same word) and re-consumes Q-1.
// ---------------------------------------------------------------------------------------------------------------
namespace b200rl {
__global__ void __launch_bounds__(256) p2p_drain_kernel(const unsigned long long* __restrict__ mailboxes, int rank, int world,
                                                        int n, unsigned int* __restrict__ state, float* __restrict__ out_mean) {
    pdl_prologue();
    const int k = threadIdx.x >> 5;
    if (k >= n) return;
    XchgArgs x{mailboxes, state, out_mean, rank, world};
    const unsigned int q = state[k];
    if (q == 0u) return;
    if (q >= 2u && state[16 + k] < q - 1u) p2p_consume_warp(x, k, q - 1u);
    __syncwarp();
    p2p_publish_warp(x, k);
    __syncwarp();
    if (state[16 + k] < q) p2p_consume_warp(x, k, q);
}
}  // namespace b200rl

extern "C" int b200rl_p2p_drain_mean(const unsigned long long* mailbox_ptrs_dev, int rank, int world, int n,
                                     unsigned int* seq_dev, float* out_mean, void* stream) {
    if (!mailbox_ptrs_dev || !seq_dev || !out_mean || n < 1 || n > b200rl::P2P_SLOT_VALS || world < 1 || world > 32 ||
        rank < 0 || rank >= world)
        return B200RL_ERR_ARG;
    return b200rl::launch_k(b200rl::p2p_drain_kernel, 1, 256, 0, (cudaStream_t)stream, mailbox_ptrs_dev, rank, world, n,
                            seq_dev, out_mean);
}
