// dist.cu -- the exchange step of the multi-GPU hot path (SURVEY.md section 8e), inside the library.
//
// One process per GPU (torchrun).  The matrix is 1-D row-block partitioned; after the local GrB_mxv every rank
// needs the other ranks' output slices (mxv: all-gather) or the monoid-fold of everybody's full-length partial
// (vxm / INP0=TRAN on a row-split A: all-reduce).  Both run as OUR kernels over NVLink/NVSwitch peer memory:
//
//   * every rank owns one cudaMalloc'd exchange region, exported with cudaIpcGetMemHandle and mapped by all
//     peers (cudaIpcOpenMemHandle): two replicated-vector buffers (values + presence bytes, double buffered),
//     one partial buffer, and a page of flags;
//   * all-gather = a push kernel (128-bit stores of the local slice straight into every rank's replicated
//     buffer at the slice's offset, system-scope fence) followed by a one-warp signal-and-wait kernel: lane p
//     raises this rank's flag in rank p (st.release.sys) and spins (ld.acquire.sys) until rank p's flag here
//     shows this step.  No host round trip, no staging copy, no NCCL call on the data path;
//   * all-reduce = publish the partial (flag), then every rank folds ITS slice of all ranks' partials with
//     peer loads in rank order (deterministic, unlike a ring) and pushes the folded slice like the all-gather.
//
// Double buffering makes the step safe without a second barrier: a rank can be at most one step ahead of a peer
// (its wait needs the peer's flag of the same step), and step t+2 writes the buffer step t used only after every
// peer has passed its own push of step t+1, i.e. after it consumed step t.
//
// The host side (pygraphblas_b200/distributed.py) only moves the 64-byte IPC handles between the processes
// (torch.distributed all_gather: control plane).
#include "common.cuh"
#include <vector>
#include <string.h>

struct B200_Comm_opaque {
    int magic; int rank, world;
    uint64_t n;                 // length of the replicated vectors
    GrB_Type type;              // type of the replicated vectors: every slice and partial must have it
    size_t esize;               // bytes per value (<= 8)
    size_t val_bytes, pres_bytes, buf_bytes, region_bytes;
    unsigned char *region = nullptr;                 // this rank's exchange region
    std::vector<unsigned char *> peer;               // every rank's region as mapped here (peer[rank] == region)
    uint64_t step = 0;                               // collectives completed (flag value of the next one = step + 1)
    GrB_Vector view = nullptr;                       // borrowed view of the current replicated buffer
    bool connected = false;
    std::string err;
};
typedef B200_Comm_opaque *B200_Comm;

static constexpr size_t FLAG_BYTES = 4096;
static constexpr int MAX_WORLD = 16;
// region layout: [buf0: values | presence][buf1: values | presence][partial: values | presence][flags: ready[16], partial_ready[16]]
static inline unsigned char *comm_buf(B200_Comm c, unsigned char *base, int which) { return base + (size_t)which * c->buf_bytes; }
static inline unsigned long long *comm_flags(B200_Comm c, unsigned char *base) { return (unsigned long long *)(base + 3 * c->buf_bytes); }

extern "C" GrB_Info GrB_Vector_new(GrB_Vector *v, GrB_Type type, GrB_Index n);
extern "C" GrB_Info GrB_Vector_free(GrB_Vector *v);

static bool comm_ok(B200_Comm c) { return c && c->magic == GB_MAGIC; }

extern "C" GrB_Info B200_Comm_create(B200_Comm *comm, int rank, int world, GrB_Index n, GrB_Type type) {
    GB_LOCK; GB_CHECK_INIT;
    if (!comm || !type) return gb_fail(GrB_NULL_POINTER, nullptr, "B200_Comm_create: NULL argument");
    if (world < 1 || world > MAX_WORLD || rank < 0 || rank >= world) return gb_fail(GrB_INVALID_VALUE, nullptr, "B200_Comm_create: rank %d of %d (at most %d ranks)", rank, world, MAX_WORLD);
    if (n == 0 || n >= ((uint64_t)1 << 31)) return gb_fail(GrB_INVALID_VALUE, nullptr, "B200_Comm_create: vector length must be in [1, 2^31)");
    if (!G.have_device) return gb_fail(GrB_PANIC, nullptr, "B200_Comm_create: no CUDA device: the exchange runs only over GPU peer memory (no CPU fallback)");
    B200_Comm c = new B200_Comm_opaque();
    c->magic = GB_MAGIC; c->rank = rank; c->world = world; c->n = n; c->type = type; c->esize = type->size;
    c->val_bytes = (((size_t)n * c->esize) + 255) & ~(size_t)255;
    c->pres_bytes = ((size_t)n + 255) & ~(size_t)255;
    c->buf_bytes = c->val_bytes + c->pres_bytes;
    c->region_bytes = 3 * c->buf_bytes + FLAG_BYTES;
    cudaError_t e = cudaMalloc((void **)&c->region, c->region_bytes);          // plain cudaMalloc: pool memory cannot be IPC-exported
    if (e != cudaSuccess) { cudaGetLastError(); delete c; return gb_fail(GrB_OUT_OF_MEMORY, nullptr, "B200_Comm_create: cudaMalloc of %zu bytes failed", c->region_bytes); }
    cudaMemsetAsync(c->region, 0, c->region_bytes, G.stream);
    cudaStreamSynchronize(G.stream);
    c->peer.assign(world, nullptr);
    c->peer[rank] = c->region;
    c->connected = world == 1;
    // the borrowed view handed out by B200_Comm_result
    GrB_Info r = GrB_Vector_new(&c->view, type, n);
    if (r != GrB_SUCCESS) { cudaFree(c->region); delete c; return r; }
    *comm = c;
    return GrB_SUCCESS;
}

extern "C" GrB_Info B200_Comm_handle(B200_Comm c, void *handle64) {
    GB_LOCK;
    if (!comm_ok(c) || !handle64) return gb_fail(GrB_NULL_POINTER, nullptr, "B200_Comm_handle: invalid argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handles are 64 bytes");
    cudaIpcMemHandle_t h;
    CU_TRY(cudaIpcGetMemHandle(&h, c->region), &c->err);
    memcpy(handle64, &h, 64);
    return GrB_SUCCESS;
}

extern "C" GrB_Info B200_Comm_connect(B200_Comm c, const void *all_handles) {
    GB_LOCK;
    if (!comm_ok(c) || !all_handles) return gb_fail(GrB_NULL_POINTER, nullptr, "B200_Comm_connect: invalid argument");
    for (int p = 0; p < c->world; ++p) {
        if (p == c->rank || c->peer[p]) continue;
        cudaIpcMemHandle_t h; memcpy(&h, (const unsigned char *)all_handles + (size_t)p * 64, 64);
        void *ptr = nullptr;
        CU_TRY(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess), &c->err);
        c->peer[p] = (unsigned char *)ptr;
    }
    c->connected = true;
    return GrB_SUCCESS;
}

extern "C" GrB_Info B200_Comm_free(B200_Comm *comm) {
    GB_LOCK;
    if (!comm || !*comm) return GrB_SUCCESS;
    B200_Comm c = *comm;
    if (!comm_ok(c)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "B200_Comm_free: invalid object");
    if (G.have_device) {
        cudaStreamSynchronize(G.stream);
        for (int p = 0; p < c->world; ++p) if (p != c->rank && c->peer[p]) cudaIpcCloseMemHandle(c->peer[p]);
        cudaFree(c->region);
    }
    GrB_Vector_free(&c->view);               // frees only what the view came to own, never the region it borrows
    c->magic = GB_FREED; delete c; *comm = nullptr;
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ kernels
struct PeerPtrs { unsigned char *p[MAX_WORLD]; };

// copy `bytes` (multiple of 16) from src to dst[peer] + off for every peer.  No flag here: the flags are raised by the NEXT kernel
// on the stream (comm_signal_wait_kernel) -- a kernel boundary orders this kernel's peer stores before it, and the per-thread
// system fence below makes that explicit.  (The first version detected its last CTA with one atomic counter: ~600 same-address
// atomics per push, 10+ us.)
__global__ void __launch_bounds__(512) comm_push_kernel(const uint4 *vsrc, size_t vbytes, size_t voff, const uint4 *psrc, size_t pbytes, size_t poff,
                                                        PeerPtrs dst, int world) {
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
    // both arrays as one sequence of 16-byte words; four words per thread and trip: the loads are issued together, then the
    // stores peer by peer (each warp writes 512 contiguous bytes per peer and word)
    const size_t nv = vbytes >> 4, np = pbytes >> 4, n = nv + np;
    for (size_t i0 = tid; i0 < n; i0 += 4 * nth) {
        uint4 v[4]; unsigned char *off[4]; bool ok[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const size_t i = i0 + (size_t)k * nth;
            ok[k] = i < n;
            const bool isv = i < nv;
            off[k] = nullptr;
            if (ok[k]) { v[k] = isv ? vsrc[i] : psrc[i - nv]; off[k] = reinterpret_cast<unsigned char *>(isv ? voff + (i << 4) : poff + ((i - nv) << 4)); }
        }
#pragma unroll 1
        for (int p = 0; p < world; ++p) {
#pragma unroll
            for (int k = 0; k < 4; ++k) if (ok[k]) *reinterpret_cast<uint4 *>(dst.p[p] + (size_t)off[k]) = v[k];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) __threadfence_system();      // cumulative over the CTA's stores (ordered before it by the barrier)
}

// the bytes after the last whole 16-byte word of each array: thread t < vtail copies value byte vsrc[t] to dst[peer] + voff + t,
// the next ptail threads presence bytes likewise.  A separate launch, only for slices that end inside a word, so that the word
// loop above stays as it was and nothing outside the slice is read or written.
__global__ void comm_push_tail_kernel(const unsigned char *vsrc, int vtail, size_t voff, const unsigned char *psrc, int ptail, size_t poff,
                                      PeerPtrs dst, int world) {
    const int t = threadIdx.x;
    if (t < vtail + ptail) {
        const bool isv = t < vtail;
        const unsigned char x = isv ? vsrc[t] : psrc[t - vtail];
        const size_t o = isv ? voff + t : poff + (t - vtail);
        for (int p = 0; p < world; ++p) dst.p[p][o] = x;
    }
    __threadfence_system();
}

// the device-wide nanosecond clock: unlike clock64 it neither depends on the SM clock nor differs between the SMs a preempted
// warp may resume on
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// one warp: lane p raises this rank's flag (slot, value `step`) in rank p's region, then waits until rank p's flag here shows `step`
__global__ void comm_signal_wait_kernel(PeerPtrs regions, size_t flag_off, const unsigned long long *my_flags, int world, int rank, int flag_slot,
                                        unsigned long long step) {
    __threadfence_system();
    if ((int)threadIdx.x < world) {
        unsigned long long *f = reinterpret_cast<unsigned long long *>(regions.p[threadIdx.x] + flag_off) + flag_slot * MAX_WORLD + rank;
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(f), "l"(step) : "memory");
        const unsigned long long *g = my_flags + flag_slot * MAX_WORLD + threadIdx.x;
        unsigned long long v;
        const unsigned long long t0 = globaltimer_ns();
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(g) : "memory");
            if (v < step && globaltimer_ns() - t0 > 20000000000ull) asm volatile("trap;");   // 20 s: a peer died -- fail loudly instead of hanging the GPU
        } while (v < step);
    }
    __syncwarp();
    __threadfence_system();
}

// fold slice [e0, e0+cnt) of every rank's partial, rank order, presence-aware; the result goes to this rank's staging slice
template <typename T>
__global__ void __launch_bounds__(256) comm_fold_kernel(PeerPtrs part, int world, size_t val_bytes, int64_t e0, int64_t cnt, int op, T *oval, uint8_t *opres) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < cnt; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = e0 + k;
        T acc = (T)0; bool has = false;
#pragma unroll 1
        for (int p = 0; p < world; ++p) {
            const uint8_t pr = reinterpret_cast<const volatile uint8_t *>(part.p[p] + val_bytes)[i];
            if (pr) {
                const T v = reinterpret_cast<const T *>(part.p[p])[i];
                acc = has ? MulApply<T, T>::f(op, acc, v) : v; has = true;      // the rule of every typed fold: OP_EQ is LXNOR
            }
        }
        oval[k] = acc; opres[k] = has;
    }
}

static inline int cgrid(size_t bytes) { return (int)std::max<size_t>(1, std::min<size_t>((bytes / 16 + 255) / 256, (size_t)G.num_sms * 4)); }
static inline int pgrid(size_t bytes) { return (int)std::max<size_t>(1, std::min<size_t>((bytes / 16 + 2047) / 2048, (size_t)G.num_sms * 2)); }

// the view borrows buffer `which`; buffers it came to own (an import into it, a write with it as output) are freed
static void comm_set_view(B200_Comm c, int which) {
    unsigned char *b = comm_buf(c, c->region, which);
    vector_adopt_device(c->view, DenseForm::borrow(b, b + c->val_bytes));
}

// flags-only round on slot `slot`: raise mine everywhere, wait for everybody's
static void comm_signal_wait(B200_Comm c, int slot, unsigned long long step) {
    PeerPtrs regions{}; for (int p = 0; p < c->world; ++p) regions.p[p] = c->peer[p];
    comm_signal_wait_kernel<<<1, 32, 0, G.stream>>>(regions, 3 * c->buf_bytes, comm_flags(c, c->region), c->world, c->rank, slot, step); GB_LAUNCHED();
}

// push (vals, pres) of `len` positions starting at row0 into buffer `which` of every rank, raise flag slot 0, wait for everybody.
// Exactly [row0, row0 + len) is written: positions no rank's slice covers keep whatever the buffer held (unspecified; zero in a
// communicator's first two collectives).
static GrB_Info comm_push_and_wait(B200_Comm c, const void *vals, const uint8_t *pres, uint64_t row0, uint64_t len, int which) {
    // non-empty slices start at multiples of 16 positions (the partition guarantees it) so that both arrays move as 16-byte words
    PeerPtrs dst{};
    for (int p = 0; p < c->world; ++p) dst.p[p] = comm_buf(c, c->peer[p], which);
    const size_t vall = (size_t)len * c->esize, vbytes = vall & ~(size_t)15, pbytes = (size_t)len & ~(size_t)15;
    const size_t voff = (size_t)row0 * c->esize, poff = c->val_bytes + (size_t)row0;
    const unsigned long long step = c->step + 1;
    if (vbytes + pbytes) { comm_push_kernel<<<pgrid(vbytes + pbytes), 512, 0, G.stream>>>((const uint4 *)vals, vbytes, voff, (const uint4 *)pres, pbytes, poff,
                                                                                        dst, c->world); GB_LAUNCHED(); }
    if (vall > vbytes || len > pbytes) {
        comm_push_tail_kernel<<<1, 32, 0, G.stream>>>((const unsigned char *)vals + vbytes, (int)(vall - vbytes), voff + vbytes, pres + pbytes, (int)(len - pbytes),
                                                      poff + pbytes, dst, c->world); GB_LAUNCHED();
    }
    comm_signal_wait(c, 0, step);
    CU_TRY(cudaGetLastError(), &c->err);
    c->step = step;
    comm_set_view(c, which);
    return GrB_SUCCESS;
}

static GrB_Info comm_check(B200_Comm c, const GrB_Vector v, const char *fn) {
    if (!comm_ok(c) || !v) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: invalid argument", fn);
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid vector", fn);
    if (!c->connected) return gb_fail(GrB_INVALID_VALUE, &c->err, "%s: B200_Comm_connect has not been called", fn);
    if (v->type->code != c->type->code) return gb_fail(GrB_DOMAIN_MISMATCH, &c->err, "%s: the vector's type does not match the communicator's", fn);
    return GrB_SUCCESS;
}

__global__ void fill_bytes_kernel(uint8_t *p, int64_t n, uint8_t v) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) p[k] = v;
}

// w_rep(row0 : row0 + slice.n) on EVERY rank = slice  (values and presence), for all ranks' slices at once
extern "C" GrB_Info B200_Comm_allgather(B200_Comm c, const GrB_Vector slice, GrB_Index row0) {
    GB_LOCK; GB_CHECK_INIT;
    GB_TRY(comm_check(c, slice, "B200_Comm_allgather"));
    // an empty slice writes nothing and is valid at any row0 <= n (equal_row_blocks starts empty trailing blocks at n)
    if (row0 + slice->n > c->n || (slice->n && (row0 & 15))) return gb_fail(GrB_INVALID_VALUE, &c->err, "B200_Comm_allgather: slice [%llu, +%llu) must lie inside the vector and, unless empty, start at a multiple of 16",
                                                            (unsigned long long)row0, (unsigned long long)slice->n);
    GbBurble burble("B200_Comm_allgather");
    GB_TRY(vector_ensure_device(slice));
    const uint8_t *pres = slice->dv.pres; DevBuf<uint8_t> ones;
    if (!pres) {                                                           // a full slice: its presence is all ones
        GB_TRY(ones.alloc((size_t)slice->n + 16, &c->err));
        fill_bytes_kernel<<<cgrid(slice->n), 256, 0, G.stream>>>(ones, (int64_t)slice->n + 16, 1); GB_LAUNCHED();
        pres = ones;
    }
    const int which = (int)((c->step + 1) & 1);
    GrB_Info r = comm_push_and_wait(c, slice->dv.val, pres, row0, slice->n, which);
    ones.reset();
    burble.note("peer push (NVLink stores) + flag wait", (double)slice->n * (c->esize + 1) * (c->world - 1));
    return r;
}

template <typename T> static void launch_fold(B200_Comm c, const PeerPtrs &part, int64_t e0, int64_t cnt, int op, void *oval, uint8_t *opres) {
    comm_fold_kernel<T><<<cgrid((size_t)cnt * 16), 256, 0, G.stream>>>(part, c->world, c->val_bytes, e0, cnt, op, (T *)oval, opres); GB_LAUNCHED();
}

// every rank contributes a full-length partial; result(i) = monoid fold, in rank order, of the partials present at i
extern "C" GrB_Info B200_Comm_allreduce(B200_Comm c, const GrB_Vector partial, GrB_Monoid monoid) {
    GB_LOCK; GB_CHECK_INIT;
    GB_TRY(comm_check(c, partial, "B200_Comm_allreduce"));
    if (!monoid || monoid->magic != GB_MAGIC) return gb_fail(GrB_NULL_POINTER, &c->err, "B200_Comm_allreduce: invalid monoid");
    if (partial->n != c->n) return gb_fail(GrB_DIMENSION_MISMATCH, &c->err, "B200_Comm_allreduce: the partial must have the communicator's length");
    const int tc = partial->type->code, op = monoid->op->opcode;
    if (monoid->op->ztype->code != tc || op == OP_USER) return gb_fail(GrB_DOMAIN_MISMATCH, &c->err, "B200_Comm_allreduce: the monoid must be a builtin one on the vector's type");
    GbBurble burble("B200_Comm_allreduce");
    GB_TRY(vector_ensure_device(partial));
    // 1. publish the partial in the exchange region and tell everybody (flag slot 1)
    unsigned char *mine = comm_buf(c, c->region, 2);
    CU_TRY(cudaMemcpyAsync(mine, partial->dv.val, (size_t)c->n * c->esize, cudaMemcpyDeviceToDevice, G.stream), &c->err);
    if (partial->dv.pres) CU_TRY(cudaMemcpyAsync(mine + c->val_bytes, partial->dv.pres, (size_t)c->n, cudaMemcpyDeviceToDevice, G.stream), &c->err);
    else { fill_bytes_kernel<<<cgrid(c->n), 256, 0, G.stream>>>(mine + c->val_bytes, (int64_t)c->n, 1); GB_LAUNCHED(); }
    const unsigned long long step = c->step + 1;
    comm_signal_wait(c, 1, step);
    // 2. fold my slice of everybody's partial (peer loads, rank order), then push it like an all-gather
    const uint64_t per = ((c->n + (uint64_t)c->world - 1) / c->world + 15) & ~(uint64_t)15;
    const uint64_t e0 = std::min<uint64_t>(c->n, per * (uint64_t)c->rank), e1 = std::min<uint64_t>(c->n, e0 + per);
    const int64_t cnt = (int64_t)(e1 - e0);
    DevBuf<void> oval; DevBuf<uint8_t> opres;
    GB_TRY(oval.alloc((size_t)cnt * c->esize + 32, &c->err));
    GB_TRY(opres.alloc((size_t)cnt + 16, &c->err));
    PeerPtrs part{}; for (int p = 0; p < c->world; ++p) part.p[p] = comm_buf(c, c->peer[p], 2);
    if (cnt > 0) switch (tc) {
        case TC_BOOL: launch_fold<bool>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_INT8: launch_fold<int8_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_INT16: launch_fold<int16_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_INT32: launch_fold<int32_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_INT64: launch_fold<int64_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_UINT8: launch_fold<uint8_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_UINT16: launch_fold<uint16_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_UINT32: launch_fold<uint32_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_UINT64: launch_fold<uint64_t>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        case TC_FP32: launch_fold<float>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
        default: launch_fold<double>(c, part, (int64_t)e0, cnt, op, oval, opres); break;
    }
    const int which = (int)(step & 1);
    GrB_Info r = comm_push_and_wait(c, oval, opres, e0, (uint64_t)cnt, which);
    oval.reset(); opres.reset();
    burble.note("peer fold (NVLink loads, rank order) + peer push + flag waits", (double)c->n * (c->esize + 1) * 2.0 * (c->world - 1) / c->world);
    return r;
}

// the replicated result of the last collective: a borrowed view, valid until the next collective on this communicator
extern "C" GrB_Info B200_Comm_result(B200_Comm c, GrB_Vector *view) {
    GB_LOCK;
    if (!comm_ok(c) || !view) return gb_fail(GrB_NULL_POINTER, nullptr, "B200_Comm_result: invalid argument");
    if (c->step == 0) comm_set_view(c, 0);
    *view = c->view;
    return GrB_SUCCESS;
}
extern "C" GrB_Info B200_Comm_barrier(B200_Comm c) {
    // an empty all-gather round: flags only (used to line the ranks up before / after a timed region)
    GB_LOCK; GB_CHECK_INIT;
    if (!comm_ok(c) || !c->connected) return gb_fail(GrB_INVALID_VALUE, nullptr, "B200_Comm_barrier: not connected");
    const unsigned long long step = c->step + 1;
    comm_signal_wait(c, 0, step);
    CU_TRY(cudaGetLastError(), &c->err);
    c->step = step;
    return GrB_SUCCESS;
}
