// exchange.cu -- K6: the repartition shuffle over peer-mapped HBM (NVLink 5 / NVSwitch), one process per GPU.
//
// Replaces TaskManager.push -> Flight do_put / do_get (pyquokka/core.py:276-376, flight.py:44-264).  Every rank owns
// a CHANNEL: a control block + a mailbox inside a symmetric allocation that all peers have mapped.  One exchange is
//
//   qk_xchg_meta   1 CTA: store my meta row (rows per destination, taken from the partition plan ON THE DEVICE, +
//                  host words: schema checksum, column widths) into every peer's control block, release a flag,
//                  spin until every peer's flag for this epoch is there, copy the meta matrix to pinned host memory.
//                  -> the only host round trip of an exchange (sizes of the receive views).
//   qk_xchg_push   the payload.  Partitioned input: ONE kernel reads each row once, orders a 2048-row tile by
//                  destination in shared memory and stores every destination's run as contiguous, coalesced
//                  stores into that peer's mailbox -- partition scatter and all-to-all fused (no local scatter, no
//                  NCCL call).  Broadcast / single-owner input: contiguous segment copies.  The last CTA releases a
//                  "data landed" flag on every peer.
//   qk_xchg_recv   1 CTA spins until every peer's data flag is there, then the mailbox columns are copied out so
//                  the mailbox can be reused.
//
// Epochs grow by one per exchange on a channel; the meta matrix is double-buffered by epoch parity.  A sender may
// write into a peer's mailbox only after it has seen that peer's meta flag for the SAME epoch, which the peer posts
// (stream order) after copying the previous epoch's rows out: the meta round is also the "mailbox free" barrier.
// Waits are single-CTA kernels, so channels used from different streams cannot starve each other, and every spin
// has a deadline (a crashed peer raises an error instead of hanging the GPU).
//
// Algorithmic bytes: payload read once locally, written once remotely (NVLink), read + written once by the copy-out.
#include "common.cuh"

namespace qk {
namespace {

constexpr int META_W = QK_XCHG_META_WORDS;

struct XchgCtrl {
    unsigned long long meta_flag[QK_MAX_PEERS];
    unsigned long long data_flag[QK_MAX_PEERS];
    unsigned long long err;                 // != 0: a wait on this rank ran past its deadline (epoch << 8 | kind)
    unsigned int push_done;                 // CTAs of the running push that have finished (last one signals)
    unsigned int pad;
    long long meta[2][QK_MAX_PEERS][META_W];
};
static_assert(sizeof(XchgCtrl) <= QK_XCHG_CTRL_BYTES, "control block size");

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// spin until *flag >= epoch; false on timeout
__device__ __forceinline__ bool wait_flag(const unsigned long long* flag, unsigned long long epoch, unsigned long long timeout_ns) {
    if (ld_acquire_sys(flag) >= epoch) return true;
    const unsigned long long t0 = globaltimer_ns();
    unsigned spins = 0;
    while (ld_acquire_sys(flag) < epoch) {
        if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > timeout_ns) return false;
        __nanosleep(64);
    }
    return true;
}

struct Chan {
    unsigned long long ctrl[QK_MAX_PEERS];
    int32_t world, me;
    unsigned long long epoch, timeout_ns;
};

struct MetaWords { long long w[META_W]; };

// ---------------------------------------------------------------- meta round
__global__ void __launch_bounds__(64) k_xchg_meta(const __grid_constant__ Chan C, const __grid_constant__ MetaWords W,
                                                  const int64_t* part_offsets, long long* out_dev, long long* out_host) {
    XchgCtrl* mine = (XchgCtrl*)C.ctrl[C.me];
    const int par = (int)(C.epoch & 1ull);
    const int t = threadIdx.x;
    if (t < META_W) {
        long long v = W.w[t];
        if (part_offsets && t < C.world) v = part_offsets[t + 1] - part_offsets[t];
        for (int p = 0; p < C.world; ++p) ((XchgCtrl*)C.ctrl[p])->meta[par][C.me][t] = v;
    }
    __threadfence_system();
    __syncthreads();
    if (t < C.world) st_release_sys(&((XchgCtrl*)C.ctrl[t])->meta_flag[C.me], C.epoch);
    bool ok = true;
    if (t < C.world) ok = wait_flag(&mine->meta_flag[t], C.epoch, C.timeout_ns);
    if (!ok) atomicExch(&mine->err, (C.epoch << 8) | 1ull);
    __syncthreads();
    __threadfence_system();
    const unsigned long long err = *(volatile unsigned long long*)&mine->err;
    for (int i = t; i < C.world * META_W; i += blockDim.x) {
        const long long v = *(volatile long long*)&mine->meta[par][i / META_W][i % META_W];
        if (out_dev) out_dev[i] = v;
        if (out_host) out_host[i] = v;
    }
    if (t == 0) {
        if (out_dev) out_dev[C.world * META_W] = (long long)err;
        if (out_host) out_host[C.world * META_W] = (long long)err;
    }
}

// ---------------------------------------------------------------- push
constexpr int X_NT = 256;
constexpr int X_TILE = 2048;             // rows per tile

constexpr int X_BUFS = QK_XCHG_MAX_BUFS;

struct PushArgs {
    const void* src[X_BUFS];
    unsigned long long dst[QK_MAX_PEERS][X_BUFS];        // peer-mapped address of the FIRST element this rank writes for (dest, column)
    long long send_lo[QK_MAX_PEERS], send_hi[QK_MAX_PEERS];   // contiguous mode: source row range per destination
    long long tile_base[QK_MAX_PEERS + 1];                    // contiguous mode: prefix sums of tiles per destination
    int8_t width[X_BUFS];                                     // element bytes
    int32_t lanes[X_BUFS];                                    // elements per row (1: scalar column)
    int32_t ncols;
};
// every buffer of an edge goes in ONE push, so that the data-landed flag is released once, after the last of them: the
// argument block is ~7 KB of __grid_constant__ parameters (sm_90 with CUDA >= 12.1 takes 32 764 bytes; 4 KB before)
static_assert(sizeof(Chan) + sizeof(PushArgs) + 3 * sizeof(void*) <= 32764, "push kernel parameters exceed 32 764 bytes");

template <class T>
__device__ __forceinline__ void copy_rows(const void* src, void* dst, long long first_row, long long r0, long long n, int lanes) {
    const T* s = (const T*)src + (first_row + r0) * lanes; T* o = (T*)dst + r0 * lanes;
    const long long m = n * lanes;
    for (long long i = threadIdx.x; i < m; i += X_NT) o[i] = s[i];
}

__device__ __forceinline__ void signal_data_landed(const Chan& C, XchgCtrl* mine) {
    // every thread's remote stores are ordered before the CTA's arrival; the last CTA to arrive releases the flags
    __threadfence_system();
    __syncthreads();
    __shared__ unsigned last;
    if (threadIdx.x == 0) last = atomicAdd(&mine->push_done, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (last) {
        __threadfence_system();
        if (threadIdx.x == 0) mine->push_done = 0;
        if ((int)threadIdx.x < C.world) st_release_sys(&((XchgCtrl*)C.ctrl[threadIdx.x])->data_flag[C.me], C.epoch);
    }
}

// contiguous segments (broadcast / single owner / pre-grouped rows): tile -> (destination, row range)
__global__ void __launch_bounds__(X_NT) k_xchg_push_contig(const __grid_constant__ Chan C, const __grid_constant__ PushArgs A) {
    XchgCtrl* mine = (XchgCtrl*)C.ctrl[C.me];
    const long long ntiles = A.tile_base[C.world];
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        int d = 0;
        while (d + 1 < C.world && tile >= A.tile_base[d + 1]) ++d;
        const long long r0 = (tile - A.tile_base[d]) * X_TILE;             // row offset inside the segment
        const long long n = min((long long)X_TILE, A.send_hi[d] - A.send_lo[d] - r0);
        for (int c = 0; c < A.ncols; ++c) {
            if (A.lanes[c] > 1 || A.width[c] == 2) {                      // vector column: whole rows, element by element
                switch (A.width[c]) {
                    case 1: copy_rows<uint8_t>(A.src[c], (void*)A.dst[d][c], A.send_lo[d], r0, n, A.lanes[c]); break;
                    case 2: copy_rows<uint16_t>(A.src[c], (void*)A.dst[d][c], A.send_lo[d], r0, n, A.lanes[c]); break;
                    case 4: copy_rows<uint32_t>(A.src[c], (void*)A.dst[d][c], A.send_lo[d], r0, n, A.lanes[c]); break;
                    default: copy_rows<uint64_t>(A.src[c], (void*)A.dst[d][c], A.send_lo[d], r0, n, A.lanes[c]); break;
                }
                continue;
            }
            switch (A.width[c]) {
                case 1: {
                    const uint8_t* s = (const uint8_t*)A.src[c] + A.send_lo[d] + r0; uint8_t* o = (uint8_t*)A.dst[d][c] + r0;
                    for (long long i = threadIdx.x; i < n; i += X_NT) o[i] = s[i];
                } break;
                case 4: {
                    const uint32_t* s = (const uint32_t*)A.src[c] + A.send_lo[d] + r0; uint32_t* o = (uint32_t*)A.dst[d][c] + r0;
                    for (long long i = threadIdx.x; i < n; i += X_NT) o[i] = s[i];
                } break;
                default: {
                    const uint64_t* s = (const uint64_t*)A.src[c] + A.send_lo[d] + r0; uint64_t* o = (uint64_t*)A.dst[d][c] + r0;
                    for (long long i = threadIdx.x; i < n; i += X_NT) o[i] = s[i];
                } break;
            }
        }
    }
    signal_data_landed(C, mine);
}

// Fused partition scatter + all-to-all.  dest[i] = position of row i in the partition-ordered output (stable plan):
// inside a tile of consecutive input rows the rows of one destination have CONSECUTIVE dest values, so after ordering
// the tile by destination in shared memory each destination's run is one contiguous, coalesced remote store.
__global__ void __launch_bounds__(X_NT) k_xchg_push_scatter(const __grid_constant__ Chan C, const __grid_constant__ PushArgs A,
                                                           const int32_t* dest, const int64_t* part_offsets, long long n) {
    XchgCtrl* mine = (XchgCtrl*)C.ctrl[C.me];
    __shared__ long long off[QK_MAX_PEERS + 1];
    __shared__ int cnt[QK_MAX_PEERS];          // rows of the tile per destination
    __shared__ int base[QK_MAX_PEERS + 1];     // their prefix sums = start of each destination's run in the ordered tile
    __shared__ long long first[QK_MAX_PEERS];  // smallest dest value of the tile per destination
    __shared__ __align__(16) unsigned char buf[X_TILE * 8];
    __shared__ unsigned short slot_of[X_TILE];  // row of the tile -> its slot in the ordered tile
    __shared__ unsigned char peer_of[X_TILE];
    if ((int)threadIdx.x <= C.world) off[threadIdx.x] = part_offsets[threadIdx.x];
    __syncthreads();
    const long long ntiles = (n + X_TILE - 1) / X_TILE;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long row0 = tile * X_TILE;
        const int m = (int)min((long long)X_TILE, n - row0);
        if ((int)threadIdx.x < C.world) { cnt[threadIdx.x] = 0; first[threadIdx.x] = 0x7fffffffffffffffLL; }
        __syncthreads();
        for (int j0 = 0; j0 < m; j0 += X_NT) {             // whole warps: the per-destination bookkeeping is warp-aggregated
            const int j = j0 + threadIdx.x;
            int p = -1;
            long long dv = 0;
            if (j < m) {
                dv = dest[row0 + j];
                p = 0;
                while (p + 1 < C.world && dv >= off[p + 1]) ++p;
                peer_of[j] = (unsigned char)p;
            }
            const unsigned peers = __match_any_sync(0xffffffffu, p);
            if (p >= 0 && (peers & lanemask_lt()) == 0) {     // lowest lane of its destination: smallest dest of the group
                atomicAdd(&cnt[p], __popc(peers));
                atomicMin((unsigned long long*)&first[p], (unsigned long long)dv);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int p = 0; p < C.world; ++p) { base[p] = s; s += cnt[p]; }
            base[C.world] = s;
        }
        __syncthreads();
        for (int j = threadIdx.x; j < m; j += X_NT) {
            const int p = peer_of[j];
            slot_of[j] = (unsigned short)(base[p] + (int)((long long)dest[row0 + j] - first[p]));
        }
        __syncthreads();
        for (int c = 0; c < A.ncols; ++c) {
            const int w = A.width[c];
            // rows -> ordered tile (shared memory)
            if (w == 8) { for (int j = threadIdx.x; j < m; j += X_NT) ((uint64_t*)buf)[slot_of[j]] = ((const uint64_t*)A.src[c])[row0 + j]; }
            else if (w == 4) { for (int j = threadIdx.x; j < m; j += X_NT) ((uint32_t*)buf)[slot_of[j]] = ((const uint32_t*)A.src[c])[row0 + j]; }
            else { for (int j = threadIdx.x; j < m; j += X_NT) buf[slot_of[j]] = ((const uint8_t*)A.src[c])[row0 + j]; }
            __syncthreads();
            // ordered tile -> the peers: slot s of destination p is row (first[p] - off[p]) + (s - base[p]) of what I send to p
            for (int s = threadIdx.x; s < m; s += X_NT) {
                int p = 0;
                while (p + 1 < C.world && s >= base[p + 1]) ++p;
                const long long r = first[p] - off[p] + (s - base[p]);
                if (w == 8) ((uint64_t*)A.dst[p][c])[r] = ((const uint64_t*)buf)[s];
                else if (w == 4) ((uint32_t*)A.dst[p][c])[r] = ((const uint32_t*)buf)[s];
                else ((uint8_t*)A.dst[p][c])[r] = buf[s];
            }
            __syncthreads();
        }
    }
    signal_data_landed(C, mine);
}

// ---------------------------------------------------------------- receive
__global__ void __launch_bounds__(32) k_xchg_wait_data(const __grid_constant__ Chan C) {
    XchgCtrl* mine = (XchgCtrl*)C.ctrl[C.me];
    if ((int)threadIdx.x < C.world && !wait_flag(&mine->data_flag[threadIdx.x], C.epoch, C.timeout_ns))
        atomicExch(&mine->err, (C.epoch << 8) | 2ull);
}

struct CopyArgs {
    const void* src[X_BUFS];
    void* dst[X_BUFS];
    long long bytes[X_BUFS];
    int32_t ncols;
};
static_assert(sizeof(CopyArgs) <= 4096, "copy-out kernel parameters");
// mailbox columns -> caller's columns (both 16-byte aligned: mailbox column bases are 256-byte aligned)
__global__ void __launch_bounds__(256) k_xchg_copy_out(const __grid_constant__ CopyArgs A) {
    for (int c = 0; c < A.ncols; ++c) {
        const long long nv = A.bytes[c] / 16;
        const uint4* s = (const uint4*)A.src[c]; uint4* d = (uint4*)A.dst[c];
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) d[i] = s[i];
        if (blockIdx.x == 0) {
            const unsigned char* sb = (const unsigned char*)A.src[c]; unsigned char* db = (unsigned char*)A.dst[c];
            for (long long i = nv * 16 + threadIdx.x; i < A.bytes[c]; i += blockDim.x) db[i] = sb[i];
        }
    }
}

int fill_chan(Chan& C, const qk_xchg* x, uint64_t epoch, const char* who) {
    if (!x) QK_FAIL(QK_ERR_INVALID, "%s: null channel", who);
    if (x->world < 1 || x->world > QK_MAX_PEERS || x->rank < 0 || x->rank >= x->world) QK_FAIL(QK_ERR_INVALID, "%s: bad world / rank", who);
    if (epoch == 0) QK_FAIL(QK_ERR_INVALID, "%s: epochs start at 1", who);
    for (int p = 0; p < x->world; ++p) {
        if (!x->ctrl[p] || (x->ctrl[p] & 15)) QK_FAIL(QK_ERR_INVALID, "%s: control block of rank %d missing / misaligned", who, p);
        C.ctrl[p] = x->ctrl[p];
    }
    C.world = x->world; C.me = x->rank; C.epoch = epoch;
    C.timeout_ns = (unsigned long long)(x->timeout_ms > 0 ? x->timeout_ms : 30000) * 1000000ull;
    return 0;
}

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_xchg_ctrl_bytes(void) { return QK_XCHG_CTRL_BYTES; }

extern "C" int qk_xchg_meta(const qk_xchg* x, uint64_t epoch, const int64_t* part_offsets, const int64_t* words,
                            int64_t* out_dev, int64_t* out_host, void* stream) {
    const char* who = "qk_xchg_meta";
    Chan C;
    if (int rc = fill_chan(C, x, epoch, who)) return rc;
    if (!words || (!out_dev && !out_host)) QK_FAIL(QK_ERR_INVALID, "%s: null words / outputs", who);
    MetaWords W;
    for (int i = 0; i < META_W; ++i) W.w[i] = words[i];
    k_xchg_meta<<<1, 64, 0, (cudaStream_t)stream>>>(C, W, part_offsets, (long long*)out_dev, (long long*)out_host);
    QK_LAUNCH_CHECK("k_xchg_meta");
    return QK_OK;
}

static int fill_push(PushArgs& A, const qk_xchg* x, const qk_column* cols, int32_t ncols, const int64_t* dst_byte_off,
                     int64_t* nrows_out, bool vectors_ok, const char* who) {
    if (ncols < 0 || ncols > QK_XCHG_MAX_BUFS) QK_FAIL(QK_ERR_INVALID, "%s: ncols out of range (%d buffers, at most %d)", who, ncols, QK_XCHG_MAX_BUFS);
    if (ncols > 0 && (!cols || !dst_byte_off)) QK_FAIL(QK_ERR_INVALID, "%s: null columns / offsets", who);
    int64_t n = ncols > 0 ? cols[0].length : 0;
    for (int c = 0; c < ncols; ++c) {
        if (int rc = vectors_ok ? check_rows_col(&cols[c], who) : check_col(&cols[c], who)) return rc;
        if (cols[c].length != n) QK_FAIL(QK_ERR_INVALID, "%s: column %d length mismatch", who, c);
        A.src[c] = cols[c].data; A.width[c] = (int8_t)dtype_size(cols[c].dtype); A.lanes[c] = row_lanes(&cols[c]);
    }
    for (int p = 0; p < x->world; ++p) {
        if (!x->mailbox[p]) QK_FAIL(QK_ERR_INVALID, "%s: mailbox of rank %d missing", who, p);
        for (int c = 0; c < ncols; ++c) {
            const int64_t o = dst_byte_off[(size_t)p * ncols + c];
            if (o < 0 || o > x->mailbox_bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: offset %lld outside the mailbox (%lld bytes)", who, (long long)o, (long long)x->mailbox_bytes);
            if (o % A.width[c]) QK_FAIL(QK_ERR_INVALID, "%s: misaligned destination offset", who);
            A.dst[p][c] = x->mailbox[p] + (unsigned long long)o;
        }
    }
    A.ncols = ncols;
    *nrows_out = n;
    return 0;
}

extern "C" int qk_xchg_push(const qk_xchg* x, uint64_t epoch, const qk_column* cols, int32_t ncols, const int64_t* send_lo,
                            const int64_t* send_hi, const int64_t* dst_byte_off, void* stream) {
    const char* who = "qk_xchg_push";
    Chan C;
    if (int rc = fill_chan(C, x, epoch, who)) return rc;
    static thread_local PushArgs A;
    int64_t n = 0;
    if (int rc = fill_push(A, x, cols, ncols, dst_byte_off, &n, true, who)) return rc;
    long long tiles = 0;
    for (int p = 0; p < x->world; ++p) {
        const int64_t lo = (ncols > 0 && send_lo) ? send_lo[p] : 0, hi = (ncols > 0 && send_hi) ? send_hi[p] : 0;
        if (lo < 0 || hi < lo || hi > n) QK_FAIL(QK_ERR_INVALID, "%s: bad row range for rank %d", who, p);
        for (int c = 0; c < ncols; ++c)
            if (dst_byte_off[(size_t)p * ncols + c] + (hi - lo) * A.width[c] * A.lanes[c] > x->mailbox_bytes)
                QK_FAIL(QK_ERR_CAPACITY, "%s: rows for rank %d do not fit its mailbox", who, p);
        A.send_lo[p] = lo; A.send_hi[p] = hi; A.tile_base[p] = tiles;
        tiles += (hi - lo + X_TILE - 1) / X_TILE;
    }
    A.tile_base[x->world] = tiles;
    k_xchg_push_contig<<<grid_size(tiles, 4, 1), X_NT, 0, (cudaStream_t)stream>>>(C, A);
    QK_LAUNCH_CHECK("k_xchg_push_contig");
    return QK_OK;
}

extern "C" int qk_xchg_push_scatter(const qk_xchg* x, uint64_t epoch, const qk_column* cols, int32_t ncols, const int32_t* dest,
                                    const int64_t* part_offsets, const int64_t* dst_byte_off, void* stream) {
    const char* who = "qk_xchg_push_scatter";
    Chan C;
    if (int rc = fill_chan(C, x, epoch, who)) return rc;
    static thread_local PushArgs A;
    int64_t n = 0;
    if (int rc = fill_push(A, x, cols, ncols, dst_byte_off, &n, false, who)) return rc;
    if (n > 0 && (!dest || !part_offsets)) QK_FAIL(QK_ERR_INVALID, "%s: null partition plan", who);
    if (n == 0) {
        for (int p = 0; p <= x->world; ++p) A.tile_base[p] = 0;
        for (int p = 0; p < x->world; ++p) A.send_lo[p] = A.send_hi[p] = 0;
        k_xchg_push_contig<<<1, X_NT, 0, (cudaStream_t)stream>>>(C, A);      // nothing to move: only the flags
        QK_LAUNCH_CHECK("k_xchg_push_contig");
        return QK_OK;
    }
    k_xchg_push_scatter<<<grid_size(n, 4, X_TILE), X_NT, 0, (cudaStream_t)stream>>>(C, A, dest, part_offsets, n);
    QK_LAUNCH_CHECK("k_xchg_push_scatter");
    return QK_OK;
}

extern "C" int qk_xchg_recv(const qk_xchg* x, uint64_t epoch, const int64_t* src_byte_off, qk_column* out, int32_t ncols, void* stream) {
    const char* who = "qk_xchg_recv";
    Chan C;
    if (int rc = fill_chan(C, x, epoch, who)) return rc;
    if (ncols < 0 || ncols > QK_XCHG_MAX_BUFS) QK_FAIL(QK_ERR_INVALID, "%s: ncols out of range (%d buffers, at most %d)", who, ncols, QK_XCHG_MAX_BUFS);
    if (ncols > 0 && (!src_byte_off || !out)) QK_FAIL(QK_ERR_INVALID, "%s: null arguments", who);
    // every argument is checked before the wait is launched: a rejected call leaves nothing on the stream
    CopyArgs A;
    long long total = 0;
    for (int c = 0; c < ncols; ++c) {
        if (int rc = check_rows_col(&out[c], who)) return rc;
        const long long bytes = out[c].length * row_bytes(&out[c]);
        if (src_byte_off[c] < 0 || (src_byte_off[c] & 15) || src_byte_off[c] + bytes > x->mailbox_bytes)
            QK_FAIL(QK_ERR_INVALID, "%s: column %d lies outside the mailbox or is misaligned", who, c);
        if (bytes > 0 && ((uintptr_t)out[c].data & 15)) QK_FAIL(QK_ERR_INVALID, "%s: output %d is not 16-byte aligned", who, c);
        A.src[c] = (const void*)(x->mailbox[x->rank] + (unsigned long long)src_byte_off[c]);
        A.dst[c] = (void*)out[c].data; A.bytes[c] = bytes;
        total += bytes;
    }
    A.ncols = ncols;
    k_xchg_wait_data<<<1, 32, 0, (cudaStream_t)stream>>>(C);
    QK_LAUNCH_CHECK("k_xchg_wait_data");
    if (total == 0) return QK_OK;
    long long nb = (total / 16 + 255) / 256 / 4 + 1;
    const long long cap = (long long)sm_count() * 8;
    if (nb > cap) nb = cap;
    k_xchg_copy_out<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(A);
    QK_LAUNCH_CHECK("k_xchg_copy_out");
    return QK_OK;
}
