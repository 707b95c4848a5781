// comm.cu -- the one collective of the path (SURVEY 8e): an all-gather of the per-shard label vectors.
//
// Rows are independent and the models are replicated, so `predict` itself never communicates: rank r classifies its
// contiguous block of ceil(n / world) rows.  Only when every rank wants the FULL label vector is there an exchange, and
// it is a single ncclAllGather of int32 class indices.  NCCL is bound at run time (dlopen of libnccl.so.2): the library
// has no link-time dependency on it, a process that never gathers never loads it, and inside a PyTorch process the
// already loaded NCCL is the one that gets used.
#include <dlfcn.h>
#include <nccl.h>   // types only; every entry point is looked up with dlsym

#include <algorithm>
#include <mutex>
#include <new>
#include <vector>

#include "common.h"

namespace tcsdn {

struct NcclApi {
    void *lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};

static NcclApi g_nccl;
static std::mutex g_nccl_mu;

static int nccl_load() {
    std::lock_guard<std::mutex> lock(g_nccl_mu);
    if (g_nccl.lib) return TCSDN_OK;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { set_error("cannot load libnccl.so.2: %s", dlerror()); return TCSDN_ECUDA; }
    NcclApi a;
    a.lib = h;
    a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(h, "ncclAllGather"));
    a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    if (!a.GetUniqueId || !a.CommInitRank || !a.AllGather || !a.CommDestroy || !a.GetErrorString) {
        set_error("libnccl.so.2 lacks an expected entry point");
        return TCSDN_ECUDA;
    }
    g_nccl = a;
    return TCSDN_OK;
}

#define TCSDN_NCCL(expr)                                                                           \
    do {                                                                                           \
        ncclResult_t _r = (expr);                                                                  \
        if (_r != ncclSuccess) {                                                                   \
            tcsdn::set_error("%s failed: %s", #expr, tcsdn::g_nccl.GetErrorString(_r));            \
            return TCSDN_ECUDA;                                                                    \
        }                                                                                          \
    } while (0)

}  // namespace tcsdn

struct tcsdn_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1;
    int32_t *d_pad = nullptr;   // staging for a short last shard (n_local < n_block)
    int64_t pad_cap = 0;
    uint8_t *d_bytes = nullptr; // byte-wide wire format: [n_block] packed local labels, then [world * n_block] gathered
    int64_t bytes_cap = 0;      // in units of n_block
    // peer-memory exchange (tcsdn_comm_gather_buffer): one allocation per rank = [world][g_block] label bytes, then 256 bytes
    // of barrier flags; g_peer[r] = rank r's allocation as seen from this process (CUDA IPC; [rank] = the local one)
    uint8_t *g_peer[tcsdn::kMaxPeers] = {nullptr};
    int64_t g_block = 0;        // bytes per rank slot (multiple of 16)
    int64_t g_bytes = 0;        // label bytes = world * g_block
};

namespace tcsdn {

// int32 labels -> one byte each (0xFF = the -1 padding of a short shard), 16 labels per thread per step
__global__ void labels_pack_u8(const int32_t *__restrict__ src, int64_t n_src, uint8_t *__restrict__ dst, int64_t n_dst) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i * 4 < n_dst; i += stride) {
        uint32_t w = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t e = i * 4 + k;
            const uint32_t v = e < n_src ? (uint32_t)src[e] & 0xFFu : 0xFFu;
            w |= v << (8 * k);
        }
        if (i * 4 + 4 <= n_dst) reinterpret_cast<uint32_t *>(dst)[i] = w;
        else for (int k = 0; i * 4 + k < n_dst; ++k) dst[i * 4 + k] = (uint8_t)(w >> (8 * k));
    }
}

__global__ void labels_unpack_u8(const uint8_t *__restrict__ src, int32_t *__restrict__ dst, int64_t n) {
    // src is 4-byte aligned (blocks start on 4-byte boundaries); dst may start at any int32 (odd block lengths): scalar stores
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i * 4 < n; i += stride) {
        if (i * 4 + 4 <= n) {
            const uint32_t w = reinterpret_cast<const uint32_t *>(src)[i];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t b = (w >> (8 * k)) & 0xFFu;
                dst[i * 4 + k] = b == 0xFFu ? -1 : (int32_t)b;
            }
        } else {
            for (int64_t e = i * 4; e < n; ++e) dst[e] = src[e] == 0xFF ? -1 : (int)src[e];
        }
    }
}

// Cross-rank barrier over peer memory.  Every rank keeps, at the end of its buffer, two flag arrays (barrier A = "I have
// entered the call", barrier B = "my label bytes are out") and a generation counter per barrier -- in DEVICE memory, so that a
// CUDA graph holding these kernels can be replayed (a generation passed as a kernel argument would be frozen at capture).
// The warp bumps the generation, writes it into slot [rank] of every rank's flag array (release, system scope: the label
// bytes this rank stored into the peers' buffers in earlier kernels of the stream are visible before the flag) and waits
// until every rank's flag in ITS OWN array has reached it (acquire).  Bounded spin: a rank that never arrives traps the
// kernel instead of hanging the GPU.
__global__ void peer_barrier_kernel(GatherOut G, int which) {
    // generations: A at +32, B at +33; ONE A and ONE B per call, both advanced by the call's B barrier (barrier A may be fused
    // into the scoring kernel, which only reads its generation)
    unsigned *ctl = G.flags[G.rank];
    const unsigned epoch = ctl[32 + which] + 1;
    if (threadIdx.x == 0) {
        __threadfence_system();
        peer_flag_arrive(G, which, epoch);
        peer_flag_wait(G, which, epoch);
        if (which == 1) { ctl[33] = epoch; ctl[32] = ctl[32] + 1; }
    }
}

__global__ void fill_bytes_kernel(GatherOut G, long long begin, long long count, unsigned char value) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count * G.world; i += (long long)gridDim.x * blockDim.x)
        G.peer[i / count][G.offset + begin + i % count] = value;
}

// int32 labels -> bytes written into slot [rank] of every rank's gathered buffer (the models without a fused store)
__global__ void scatter_labels_kernel(GatherOut G, const int32_t *__restrict__ labels, long long n) {
    const long long n16 = (n + 15) / 16;
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < n16; c += (long long)gridDim.x * blockDim.x) {
        uint32_t w[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const long long e = c * 16 + k;
            if (e < n) w[k >> 2] = (w[k >> 2] & ~(0xFFu << (8 * (k & 3)))) | (((uint32_t)labels[e] & 0xFFu) << (8 * (k & 3)));
        }
        const uint4 v = make_uint4(w[0], w[1], w[2], w[3]);
        for (int pr = 0; pr < G.world; ++pr) *reinterpret_cast<uint4 *>(G.peer[pr] + G.offset + c * 16) = v;
    }
}

}  // namespace tcsdn

using namespace tcsdn;

extern "C" {

int tcsdn_comm_unique_id(void *id_out) {
    if (!id_out) { set_error("comm_unique_id: NULL output"); return TCSDN_EINVAL; }
    TCSDN_TRY(nccl_load());
    ncclUniqueId id;
    TCSDN_NCCL(g_nccl.GetUniqueId(&id));
    static_assert(sizeof(ncclUniqueId) == TCSDN_COMM_ID_BYTES, "ncclUniqueId size");
    memcpy(id_out, &id, sizeof(id));
    return TCSDN_OK;
}

int tcsdn_comm_init(int32_t rank, int32_t world, const void *unique_id, tcsdn_comm_t **out) {
    if (!out || !unique_id || world < 1 || rank < 0 || rank >= world) {
        set_error("comm_init: bad arguments (rank %d of %d)", rank, world);
        return TCSDN_EINVAL;
    }
    *out = nullptr;
    TCSDN_TRY(nccl_load());
    ncclUniqueId id;
    memcpy(&id, unique_id, sizeof(id));
    tcsdn_comm *c = new (std::nothrow) tcsdn_comm();
    if (!c) { set_error("comm_init: out of memory"); return TCSDN_ENOMEM; }
    c->rank = rank; c->world = world;
    ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, id, rank);
    if (r != ncclSuccess) {
        set_error("ncclCommInitRank failed: %s", g_nccl.GetErrorString(r));
        delete c;
        return TCSDN_ECUDA;
    }
    *out = c;
    return TCSDN_OK;
}

int tcsdn_allgather_labels(tcsdn_comm_t *c, const int32_t *local, int64_t n_local, int64_t n_block, int32_t *all,
                           void *cuda_stream) {
    if (!c || !all || n_block < 0 || n_local < 0 || n_local > n_block || (n_local > 0 && !local)) {
        set_error("allgather_labels: bad arguments");
        return TCSDN_EINVAL;
    }
    if (n_block == 0) return TCSDN_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    const int32_t *send = local;
    if (n_local < n_block) {   // short (or empty) last shard: pad with -1 so that every rank contributes n_block entries
        if (c->pad_cap < n_block) {
            if (c->d_pad) cudaFree(c->d_pad);
            c->d_pad = nullptr; c->pad_cap = 0;
            TCSDN_CUDA(cudaMalloc(&c->d_pad, (size_t)n_block * sizeof(int32_t)));
            c->pad_cap = n_block;
        }
        TCSDN_CUDA(cudaMemsetAsync(c->d_pad, 0xFF, (size_t)n_block * sizeof(int32_t), st));
        if (n_local > 0)
            TCSDN_CUDA(cudaMemcpyAsync(c->d_pad, local, (size_t)n_local * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
        send = c->d_pad;
    }
    TCSDN_NCCL(g_nccl.AllGather(send, all, (size_t)n_block, ncclInt32, c->comm, st));
    return TCSDN_OK;
}

// Same result, a quarter of the bytes on the wire: class indices below 255 travel as one byte each (SURVEY 8e); every rank
// packs its block, one ncclAllGather of bytes, every rank widens the gathered vector back to int32.  Everything is
// enqueued on `cuda_stream` with no host synchronisation, so predict + gather can be captured into one CUDA graph
// (staging buffers are sized on the first call with a given n_block: make that call outside the capture).
int tcsdn_allgather_labels_u8(tcsdn_comm_t *c, const int32_t *local, int64_t n_local, int64_t n_block, int32_t *all,
                              int32_t n_classes, void *cuda_stream) {
    if (!c || !all || n_block < 0 || n_local < 0 || n_local > n_block || (n_local > 0 && !local)) {
        set_error("allgather_labels_u8: bad arguments");
        return TCSDN_EINVAL;
    }
    if (n_classes < 1 || n_classes > 255) return tcsdn_allgather_labels(c, local, n_local, n_block, all, cuda_stream);
    if (n_block == 0) return TCSDN_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    const int64_t nb4 = (n_block + 3) & ~(int64_t)3;   // blocks start on 4-byte boundaries
    if (c->bytes_cap < nb4) {
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cap);
        if (cap != cudaStreamCaptureStatusNone) {
            set_error("allgather_labels_u8: the first call with n_block=%lld allocates staging memory; make it outside the graph capture", (long long)n_block);
            return TCSDN_EINVAL;
        }
        if (c->d_bytes) cudaFree(c->d_bytes);
        c->d_bytes = nullptr; c->bytes_cap = 0;
        TCSDN_CUDA(cudaMalloc(&c->d_bytes, (size_t)nb4 * (size_t)(c->world + 1)));
        c->bytes_cap = nb4;
    }
    uint8_t *mine = c->d_bytes, *gathered = c->d_bytes + c->bytes_cap;
    const int threads = 256;
    int64_t blocks = (nb4 / 4 + threads - 1) / threads;
    if (blocks > 132 * 8) blocks = 132 * 8;
    labels_pack_u8<<<(unsigned)blocks, threads, 0, st>>>(local, n_local, mine, nb4);
    TCSDN_CUDA(cudaGetLastError());
    TCSDN_NCCL(g_nccl.AllGather(mine, gathered, (size_t)nb4, ncclUint8, c->comm, st));
    if (nb4 == n_block) {
        const int64_t total = n_block * c->world;
        blocks = (total / 4 + threads - 1) / threads;
        if (blocks > 132 * 8) blocks = 132 * 8;
        labels_unpack_u8<<<(unsigned)blocks, threads, 0, st>>>(gathered, all, total);
    } else {
        for (int r = 0; r < c->world; ++r)   // odd block length: per-rank segments (destination blocks are n_block apart)
            labels_unpack_u8<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(blocks, 132 * 8)), threads, 0, st>>>(
                gathered + (size_t)r * nb4, all + (size_t)r * n_block, n_block);
    }
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

/* ---- peer-memory exchange: the gathered label vector is written by the classification kernels themselves --------------- */

static void gather_release(tcsdn_comm *c) {
    for (int r = 0; r < c->world && r < kMaxPeers; ++r) {
        if (!c->g_peer[r]) continue;
        if (r == c->rank) cudaFree(c->g_peer[r]); else cudaIpcCloseMemHandle(c->g_peer[r]);
        c->g_peer[r] = nullptr;
    }
    c->g_block = c->g_bytes = 0;
}

int tcsdn_comm_gather_buffer(tcsdn_comm_t *c, int64_t n_block, const uint8_t **gathered_out, int64_t *slot_bytes_out) {
    if (!c || n_block < 0) { set_error("comm_gather_buffer: bad arguments"); return TCSDN_EINVAL; }
    if (c->world > kMaxPeers) { set_error("comm_gather_buffer: at most %d ranks (one NVSwitch domain)", kMaxPeers); return TCSDN_EINVAL; }
    const int64_t blk = (n_block + 15) & ~(int64_t)15;
    if (c->g_block < blk) {   // collective (re)allocation: every rank calls with the same n_block
        cudaDeviceSynchronize();
        gather_release(c);
        const size_t label_bytes = (size_t)blk * c->world;
        const size_t total = label_bytes + 256;                         // labels, then the barrier flags (zeroed)
        uint8_t *mine = nullptr;
        TCSDN_CUDA(cudaMalloc(&mine, total));
        TCSDN_CUDA(cudaMemset(mine, 0xFF, label_bytes));
        TCSDN_CUDA(cudaMemset(mine + label_bytes, 0, 256));
        c->g_peer[c->rank] = mine;
        c->g_block = blk; c->g_bytes = (int64_t)label_bytes;
        if (c->world > 1) {
            // exchange the CUDA IPC handles through the communicator itself (64 bytes per rank)
            cudaIpcMemHandle_t h;
            TCSDN_CUDA(cudaIpcGetMemHandle(&h, mine));
            uint8_t *d_h = nullptr;
            TCSDN_CUDA(cudaMalloc(&d_h, sizeof(h) * (size_t)(c->world + 1)));
            TCSDN_CUDA(cudaMemcpy(d_h, &h, sizeof(h), cudaMemcpyHostToDevice));
            ncclResult_t nr = g_nccl.AllGather(d_h, d_h + sizeof(h), sizeof(h), ncclUint8, c->comm, nullptr);
            if (nr != ncclSuccess) { cudaFree(d_h); set_error("ncclAllGather(ipc handles) failed: %s", g_nccl.GetErrorString(nr)); return TCSDN_ECUDA; }
            std::vector<cudaIpcMemHandle_t> all((size_t)c->world);
            cudaError_t e = cudaMemcpy(all.data(), d_h + sizeof(h), sizeof(h) * (size_t)c->world, cudaMemcpyDeviceToHost);   // synchronises
            cudaFree(d_h);
            if (e != cudaSuccess) { set_error("ipc handle exchange failed: %s", cudaGetErrorString(e)); return TCSDN_ECUDA; }
            for (int r = 0; r < c->world; ++r) {
                if (r == c->rank) continue;
                void *p = nullptr;
                e = cudaIpcOpenMemHandle(&p, all[(size_t)r], cudaIpcMemLazyEnablePeerAccess);
                if (e != cudaSuccess) { set_error("cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e)); return TCSDN_ECUDA; }
                c->g_peer[r] = static_cast<uint8_t *>(p);
            }
        }
    }
    if (gathered_out) *gathered_out = c->g_peer[c->rank];
    if (slot_bytes_out) *slot_bytes_out = c->g_block;
    return TCSDN_OK;
}

int tcsdn_predict_gathered(tcsdn_model_t *m, tcsdn_comm_t *c, const void *x, int64_t n_local, int32_t d, int32_t x_dtype,
                           const uint8_t **gathered_out, void *cuda_stream) {
    if (!m || !c || n_local < 0 || (n_local > 0 && !x)) { set_error("predict_gathered: bad arguments"); return TCSDN_EINVAL; }
    if (d != m->d) { set_error("X has %d features, but the model is expecting %d features as input", d, m->d); return TCSDN_EINVAL; }
    if (x_dtype != TCSDN_F32 && x_dtype != TCSDN_F64) { set_error("x_dtype must be TCSDN_F32 or TCSDN_F64"); return TCSDN_EINVAL; }
    if (m->n_classes > 255 && m->kind != TCSDN_KIND_FOREST && m->kind != TCSDN_KIND_KNN && m->kind != TCSDN_KIND_SVC) {
        set_error("predict_gathered: labels travel as bytes, the model has %d classes", m->n_classes); return TCSDN_EINVAL; }
    if (!c->g_peer[c->rank] || n_local > c->g_block) { set_error("predict_gathered: call tcsdn_comm_gather_buffer(n_block >= %lld) first", (long long)n_local); return TCSDN_EINVAL; }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    GatherOut G;
    memset(&G, 0, sizeof(G));
    G.world = c->world; G.rank = c->rank;
    G.slot = c->g_block;
    G.offset = (long long)c->rank * c->g_block;
    for (int r = 0; r < c->world; ++r) {
        G.peer[r] = c->g_peer[r];
        G.flags[r] = reinterpret_cast<unsigned *>(c->g_peer[r] + (size_t)c->g_bytes);   // the barrier words behind the labels
    }
    const bool fused = n_local > 0 && (m->kind == TCSDN_KIND_LINEAR || m->kind == TCSDN_KIND_GNB || m->kind == TCSDN_KIND_KMEANS) &&
                       x_dtype == TCSDN_F32 && m->sp_valid && (m->d == 4 || m->d == 8 || m->d == 12 || m->d == 16) &&
                       (reinterpret_cast<uintptr_t>(x) & 15) == 0 && m->opt_engine != 1;
    if (fused) {
        // ONE kernel classifies and gathers: it arrives at barrier A when it starts, every CTA waits for A before its first store
        // into the peers, and stores each label byte into all ranks' buffers (scorers.cu); then the one-warp barrier B
        TCSDN_TRY(launch_scorer(m, x, n_local, x_dtype, nullptr, nullptr, m->opt_check_finite ? m->d_flag : nullptr, st, &G));
        const int64_t d16 = (n_local + 15) & ~(int64_t)15;
        if (d16 < c->g_block) fill_bytes_kernel<<<8, 256, 0, st>>>(G, d16, c->g_block - d16, 0xFF);
        peer_barrier_kernel<<<1, 32, 0, st>>>(G, 1);
        TCSDN_CUDA(cudaGetLastError());
        if (gathered_out) *gathered_out = c->g_peer[c->rank];
        return TCSDN_OK;
    }
    // The other estimators: their own kernels into a local int32 vector first (no peer is touched), then barrier A -- no rank
    // stores a label of this call before every rank has ENTERED the call, i.e. before everything the others enqueued behind
    // their previous call (the readers of the previous vector) has run --, one scatter kernel over peer memory, barrier B.
    if (n_local > 0) {
        if (c->pad_cap < n_local) {
            cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
            cudaStreamIsCapturing(st, &cap);
            if (cap != cudaStreamCaptureStatusNone) { set_error("predict_gathered: first call allocates; make it outside the graph capture"); return TCSDN_EINVAL; }
            if (c->d_pad) cudaFree(c->d_pad);
            c->d_pad = nullptr; c->pad_cap = 0;
            TCSDN_CUDA(cudaMalloc(&c->d_pad, (size_t)c->g_block * sizeof(int32_t)));
            c->pad_cap = c->g_block;
        }
        TCSDN_TRY(tcsdn_predict(m, x, n_local, d, x_dtype, TCSDN_DEVICE, c->d_pad, nullptr, cuda_stream));
    }
    peer_barrier_kernel<<<1, 32, 0, st>>>(G, 0);
    if (n_local > 0) {
        int64_t blocks = ((n_local + 15) / 16 + 255) / 256;
        if (blocks > 132 * 4) blocks = 132 * 4;
        scatter_labels_kernel<<<(unsigned)blocks, 256, 0, st>>>(G, c->d_pad, n_local);
    }
    const int64_t done16 = (n_local + 15) & ~(int64_t)15;
    if (done16 < c->g_block)   // a short block: the rest of the slot reads -1 (0xFF) on every rank
        fill_bytes_kernel<<<8, 256, 0, st>>>(G, done16, c->g_block - done16, 0xFF);
    peer_barrier_kernel<<<1, 32, 0, st>>>(G, 1);   // everybody's bytes have landed when it retires
    TCSDN_CUDA(cudaGetLastError());
    if (gathered_out) *gathered_out = c->g_peer[c->rank];
    return TCSDN_OK;
}

void tcsdn_comm_destroy(tcsdn_comm_t *c) {
    if (!c) return;
    gather_release(c);
    if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
    if (c->d_pad) cudaFree(c->d_pad);
    if (c->d_bytes) cudaFree(c->d_bytes);
    delete c;
}

}  // extern "C"
