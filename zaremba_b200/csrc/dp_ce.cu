// Data-parallel gradient all-reduce over NVLink peer memory WITHOUT using SMs for the transport.
//
// Why not NCCL here: the backward recurrence is a 128-CTA cluster kernel that needs (almost) every SM
// co-resident; an NCCL all-reduce running next to it takes 24 SMs (NVLS channels), the cluster kernel can
// no longer be fully resident and stalls at its grid barrier (measured: rec_bwd 0.53 -> 1.06 ms, step
// 2.43 -> 2.67 ms at N=8).  Copy engines move peer memory without touching the SMs, so the reduction of a
// finished gradient bucket can run underneath the rest of backward.
//
// One process per GPU.  The flat gradient buffer and a small flag block are allocated here with cudaMalloc
// and exported through CUDA IPC; every rank maps every peer.  Per bucket [lo,hi), split into `world` shards:
//   ready      compute stream, after the bucket's gradients are complete: ONE cuStreamWriteValue32 of a
//              sequence number into the rank's own flag block (peers poll it through the IPC mapping)
//   scatter    per peer p, on its own stream (copies from different peers run on different copy engines):
//              cuStreamWaitValue32(ready[p]) ; cudaMemcpyAsync(staging[p] <- peer p's copy of MY shard)
//   reduce     a small kernel sums the world-1 staged slices into my shard of g (fixed rank order:
//              deterministic, same bits on every rank) ; "reduced" flag to every peer
//   gather     per peer p: wait reduced[p] ; cudaMemcpyAsync(g[shard p] <- peer p's g[shard p])
//   done       flag to every peer; the next step's first write into g waits for all peers' done flags
//              (they pulled my reduced shard out of my g).
// The data path is a reduce-scatter followed by an all-gather: 2*(world-1)/world * bytes over NVLink per GPU,
// the same volume as a ring all-reduce.
#include <string.h>

#include <vector>

#include <cuda.h>

#include "engine.h"

struct zrb_dp {
    int rank = 0, world = 1;
    float* g = nullptr;            // flat gradient buffer (owned)
    int64_t n = 0;
    uint32_t* flags = nullptr;     // [3][kMaxBuckets] ready / reduced / done: written locally, polled by peers (owned)
    float* staging = nullptr;      // [world-1][max_shard]
    int64_t max_shard = 0;
    std::vector<float*> peer_g;    // mapped peer gradient buffers (peer_g[rank] = g)
    std::vector<uint32_t*> peer_flags;
    int spp = 1;                          // copy streams per peer (each stream is served by a copy engine)
    std::vector<cudaStream_t> streams;   // [world][spp]
    cudaStream_t reduce_stream = nullptr;
    std::vector<cudaEvent_t> ev_copy;    // [world][spp]
    cudaEvent_t ev_reduced = nullptr, ev_done = nullptr, ev_ready = nullptr;
    uint32_t seq = 0;              // sequence number of the bucket being reduced
    uint32_t last_done_seq = 0;
    bool imported = false;
};

namespace zrb {

constexpr int kMaxBuckets = 16;

typedef CUresult (*StreamValFn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static StreamValFn g_wait32 = nullptr, g_write32 = nullptr;

static int load_stream_memops() {
    if (g_wait32 && g_write32) return ZRB_OK;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
        set_error("cuStreamWaitValue32 not available");
        return ZRB_E_CUDA;
    }
    g_wait32 = (StreamValFn)p;
    if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
        set_error("cuStreamWriteValue32 not available");
        return ZRB_E_CUDA;
    }
    g_write32 = (StreamValFn)p;
    return ZRB_OK;
}

#define ZRB_CU(call)                                                                      \
    do {                                                                                  \
        CUresult r_ = (call);                                                             \
        if (r_ != CUDA_SUCCESS) {                                                         \
            zrb::set_error("%s:%d %s -> CUresult %d", __FILE__, __LINE__, #call, (int)r_); \
            return ZRB_E_CUDA;                                                            \
        }                                                                                 \
    } while (0)

// dst[i] += sum_p src_p[i]   (p in fixed order), 16-byte vectors
__global__ void dp_reduce_kernel(float* __restrict__ dst, const float* __restrict__ staging, int64_t stride, int nsrc,
                                 int64_t n) {
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 a = reinterpret_cast<float4*>(dst)[i];
        for (int p = 0; p < nsrc; ++p) {
            float4 b = __ldcs(reinterpret_cast<const float4*>(staging + p * stride) + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        reinterpret_cast<float4*>(dst)[i] = a;
    }
    for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x) {
        float a = dst[i];
        for (int p = 0; p < nsrc; ++p) a += staging[p * stride + i];
        dst[i] = a;
    }
}

// flag of `kind` (0 ready, 1 reduced, 2 done) for bucket b inside a rank's flag block.  Every rank writes only
// its OWN block (one stream write per event instead of one per peer) and waits on the peers' blocks through the
// IPC mapping.
static uint32_t* flag_ptr(uint32_t* base, int kind, int bucket) { return base + (size_t)kind * kMaxBuckets + bucket; }

}  // namespace zrb

using namespace zrb;

extern "C" {

int zrb_dp_create(int32_t rank, int32_t world, int64_t n_grad, zrb_dp** out) {
    ZRB_REQUIRE(out && world >= 1 && rank >= 0 && rank < world && n_grad > 0, "bad arguments");
    ZRB_TRY(load_stream_memops());
    zrb_dp* d = new zrb_dp();
    d->rank = rank; d->world = world; d->n = n_grad;
    d->max_shard = ((n_grad + world - 1) / world + 3) & ~(int64_t)3;
    ZRB_CUDA(cudaMalloc(&d->g, (size_t)n_grad * sizeof(float)));
    ZRB_CUDA(cudaMemset(d->g, 0, (size_t)n_grad * sizeof(float)));
    ZRB_CUDA(cudaMalloc(&d->flags, (size_t)3 * kMaxBuckets * sizeof(uint32_t)));
    ZRB_CUDA(cudaMemset(d->flags, 0, (size_t)3 * kMaxBuckets * sizeof(uint32_t)));
    if (world > 1) ZRB_CUDA(cudaMalloc(&d->staging, (size_t)(world - 1) * d->max_shard * sizeof(float)));
    d->peer_g.assign(world, nullptr);
    d->peer_flags.assign(world, nullptr);
    d->peer_g[rank] = d->g;
    d->peer_flags[rank] = d->flags;
    d->spp = 1;   // measured: one stream per peer already runs at 680 GB/s, more streams are slower
    for (int i = 0; i < world * d->spp; ++i) {
        cudaStream_t s;
        ZRB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        d->streams.push_back(s);
        cudaEvent_t e;
        ZRB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        d->ev_copy.push_back(e);
    }
    ZRB_CUDA(cudaStreamCreateWithFlags(&d->reduce_stream, cudaStreamNonBlocking));
    ZRB_CUDA(cudaEventCreateWithFlags(&d->ev_reduced, cudaEventDisableTiming));
    ZRB_CUDA(cudaEventCreateWithFlags(&d->ev_done, cudaEventDisableTiming));
    ZRB_CUDA(cudaEventCreateWithFlags(&d->ev_ready, cudaEventDisableTiming));
    *out = d;
    return ZRB_OK;
}

void zrb_dp_destroy(zrb_dp* d) {
    if (!d) return;
    cudaDeviceSynchronize();
    for (int p = 0; p < d->world; ++p) {
        if (p == d->rank) continue;
        if (d->peer_g[p]) cudaIpcCloseMemHandle(d->peer_g[p]);
        if (d->peer_flags[p]) cudaIpcCloseMemHandle(d->peer_flags[p]);
    }
    for (auto s : d->streams) cudaStreamDestroy(s);
    for (auto e : d->ev_copy) cudaEventDestroy(e);
    if (d->reduce_stream) cudaStreamDestroy(d->reduce_stream);
    if (d->ev_reduced) cudaEventDestroy(d->ev_reduced);
    if (d->ev_done) cudaEventDestroy(d->ev_done);
    if (d->ev_ready) cudaEventDestroy(d->ev_ready);
    cudaFree(d->g); cudaFree(d->flags); cudaFree(d->staging);
    delete d;
}

float* zrb_dp_grad_buffer(zrb_dp* d) { return d ? d->g : nullptr; }

// 128-byte blob: IPC handles of the gradient buffer and of the flag block
int zrb_dp_export(zrb_dp* d, void* h_blob128) {
    ZRB_REQUIRE(d && h_blob128, "null argument");
    cudaIpcMemHandle_t hg, hf;
    ZRB_CUDA(cudaIpcGetMemHandle(&hg, d->g));
    ZRB_CUDA(cudaIpcGetMemHandle(&hf, d->flags));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "unexpected IPC handle size");
    memcpy(h_blob128, &hg, 64);
    memcpy((char*)h_blob128 + 64, &hf, 64);
    return ZRB_OK;
}

// h_blobs: world x 128 bytes, in rank order (as all-gathered by the host)
int zrb_dp_import(zrb_dp* d, const void* h_blobs) {
    ZRB_REQUIRE(d && h_blobs, "null argument");
    for (int p = 0; p < d->world; ++p) {
        if (p == d->rank) continue;
        cudaIpcMemHandle_t hg, hf;
        memcpy(&hg, (const char*)h_blobs + (size_t)p * 128, 64);
        memcpy(&hf, (const char*)h_blobs + (size_t)p * 128 + 64, 64);
        void* pg = nullptr; void* pf = nullptr;
        ZRB_CUDA(cudaIpcOpenMemHandle(&pg, hg, cudaIpcMemLazyEnablePeerAccess));
        ZRB_CUDA(cudaIpcOpenMemHandle(&pf, hf, cudaIpcMemLazyEnablePeerAccess));
        d->peer_g[p] = (float*)pg;
        d->peer_flags[p] = (uint32_t*)pf;
    }
    d->imported = true;
    return ZRB_OK;
}

// Before the first write of a new step into g: every peer must have pulled my reduced shards of the previous step.
int zrb_dp_begin_step(zrb_dp* d, void* compute_stream) {
    ZRB_REQUIRE(d, "null argument");
    if (d->world == 1 || d->last_done_seq == 0) return ZRB_OK;
    cudaStream_t rs = d->reduce_stream;
    for (int p = 0; p < d->world; ++p) {
        if (p == d->rank) continue;
        ZRB_CU(g_wait32((CUstream)rs, (CUdeviceptr)flag_ptr(d->peer_flags[p], 2, 0), d->last_done_seq,
                        CU_STREAM_WAIT_VALUE_GEQ));
    }
    ZRB_CUDA(cudaEventRecord(d->ev_done, rs));
    ZRB_CUDA(cudaStreamWaitEvent((cudaStream_t)compute_stream, d->ev_done, 0));
    return ZRB_OK;
}

// Make `compute_stream` wait for every bucket reduction enqueued so far in this step and publish "done".
int zrb_dp_finish_step(zrb_dp* d, void* compute_stream) {
    ZRB_REQUIRE(d, "null argument");
    const int W = d->world, R = d->rank;
    if (W == 1 || d->seq == d->last_done_seq) return ZRB_OK;
    cudaStream_t rs = d->reduce_stream, cs = (cudaStream_t)compute_stream;
    const uint32_t seq = d->seq;
    ZRB_CUDA(cudaStreamWaitEvent(rs, d->ev_reduced, 0));
    for (int p = 0; p < W; ++p)
        if (p != R)
            for (int c = 0; c < d->spp; ++c) ZRB_CUDA(cudaStreamWaitEvent(rs, d->ev_copy[p * d->spp + c], 0));
    ZRB_CU(g_write32((CUstream)rs, (CUdeviceptr)flag_ptr(d->flags, 2, 0), seq, 0));
    ZRB_CUDA(cudaEventRecord(d->ev_done, rs));
    ZRB_CUDA(cudaStreamWaitEvent(cs, d->ev_done, 0));
    d->last_done_seq = seq;
    return ZRB_OK;
}

// Bucket `b` of this step covers g[lo, hi) and is complete on `compute_stream`.  Enqueues the whole reduce-scatter +
// all-gather of the bucket on internal streams; nothing blocks the host.  `last` marks the final bucket of the step.
int zrb_dp_allreduce_bucket(zrb_dp* d, int32_t b, int64_t lo, int64_t hi, int32_t last, void* compute_stream) {
    ZRB_REQUIRE(d && d->imported && b >= 0 && b < kMaxBuckets && lo >= 0 && hi <= d->n && lo < hi, "bad bucket");
    const int W = d->world, R = d->rank;
    if (W == 1) return ZRB_OK;
    const uint32_t seq = ++d->seq;
    cudaStream_t cs = (cudaStream_t)compute_stream;
    const int64_t nb = hi - lo;
    int64_t shard = ((nb + W - 1) / W + 3) & ~(int64_t)3;
    auto s_lo = [&](int r) { return lo + (int64_t)r * shard < hi ? lo + (int64_t)r * shard : hi; };
    auto s_hi = [&](int r) { return lo + (int64_t)(r + 1) * shard < hi ? lo + (int64_t)(r + 1) * shard : hi; };

    // ready: after the bucket's last kernel on the compute stream, tell every peer
    ZRB_CU(g_write32((CUstream)cs, (CUdeviceptr)flag_ptr(d->flags, 0, b), seq, 0));
    ZRB_CUDA(cudaEventRecord(d->ev_ready, cs));

    // scatter phase: pull my shard of every peer's bucket (one stream per peer -> independent copy engines)
    const int64_t my_lo = s_lo(R), my_n = s_hi(R) - s_lo(R);
    int slot = 0;
    for (int p = 0; p < W; ++p) {
        if (p == R) continue;
        const int64_t piece = ((my_n + d->spp - 1) / d->spp + 3) & ~(int64_t)3;
        for (int c = 0; c < d->spp; ++c) {
            cudaStream_t st = d->streams[p * d->spp + c];
            // the staging slot is reused by every bucket: the previous bucket's reduce kernel must have read it
            ZRB_CUDA(cudaStreamWaitEvent(st, d->ev_reduced, 0));
            ZRB_CU(g_wait32((CUstream)st, (CUdeviceptr)flag_ptr(d->peer_flags[p], 0, b), seq, CU_STREAM_WAIT_VALUE_GEQ));
            const int64_t o = (int64_t)c * piece, cnt = o < my_n ? (my_n - o < piece ? my_n - o : piece) : 0;
            if (cnt > 0)
                ZRB_CUDA(cudaMemcpyAsync(d->staging + (size_t)slot * d->max_shard + o, d->peer_g[p] + my_lo + o,
                                         (size_t)cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
            ZRB_CUDA(cudaEventRecord(d->ev_copy[p * d->spp + c], st));
        }
        ++slot;
    }
    // reduce: my own bucket must be complete too (ev_ready), then sum the staged slices in rank order
    cudaStream_t rs = d->reduce_stream;
    ZRB_CUDA(cudaStreamWaitEvent(rs, d->ev_ready, 0));
    for (int p = 0; p < W; ++p)
        if (p != R)
            for (int c = 0; c < d->spp; ++c) ZRB_CUDA(cudaStreamWaitEvent(rs, d->ev_copy[p * d->spp + c], 0));
    if (my_n > 0) {
        int blocks = (int)((my_n / 4 + 255) / 256);
        if (blocks > 64) blocks = 64;      // small on purpose: shares the SMs with the persistent kernels
        if (blocks < 1) blocks = 1;
        dp_reduce_kernel<<<blocks, 256, 0, rs>>>(d->g + my_lo, d->staging, d->max_shard, W - 1, my_n);
        ZRB_KERNEL_CHECK();
    }
    ZRB_CU(g_write32((CUstream)rs, (CUdeviceptr)flag_ptr(d->flags, 1, b), seq, 0));
    ZRB_CUDA(cudaEventRecord(d->ev_reduced, rs));

    // gather phase: pull every peer's reduced shard into my g
    for (int p = 0; p < W; ++p) {
        if (p == R) continue;
        const int64_t pl = s_lo(p), pn = s_hi(p) - s_lo(p);
        const int64_t piece = ((pn + d->spp - 1) / d->spp + 3) & ~(int64_t)3;
        for (int c = 0; c < d->spp; ++c) {
            cudaStream_t st = d->streams[p * d->spp + c];
            ZRB_CU(g_wait32((CUstream)st, (CUdeviceptr)flag_ptr(d->peer_flags[p], 1, b), seq, CU_STREAM_WAIT_VALUE_GEQ));
            const int64_t o = (int64_t)c * piece, cnt = o < pn ? (pn - o < piece ? pn - o : piece) : 0;
            if (cnt > 0)
                ZRB_CUDA(cudaMemcpyAsync(d->g + pl + o, d->peer_g[p] + pl + o, (size_t)cnt * sizeof(float),
                                         cudaMemcpyDeviceToDevice, st));
            ZRB_CUDA(cudaEventRecord(d->ev_copy[p * d->spp + c], st));
        }
    }
    if (last) {
        // join everything of this step on the reduce stream, publish "done", and let the compute stream continue
        ZRB_CUDA(cudaStreamWaitEvent(rs, d->ev_reduced, 0));
        for (int p = 0; p < W; ++p)
            if (p != R)
                for (int c = 0; c < d->spp; ++c) ZRB_CUDA(cudaStreamWaitEvent(rs, d->ev_copy[p * d->spp + c], 0));
        ZRB_CU(g_write32((CUstream)rs, (CUdeviceptr)flag_ptr(d->flags, 2, 0), seq, 0));
        ZRB_CUDA(cudaEventRecord(d->ev_done, rs));
        ZRB_CUDA(cudaStreamWaitEvent(cs, d->ev_done, 0));
        d->last_done_seq = seq;
    }
    return ZRB_OK;
}

}  // extern "C"
