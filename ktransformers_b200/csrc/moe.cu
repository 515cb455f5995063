// Routed experts, dense linear and gated MLP on the streaming integer GEMV kernels (gemv.cuh).
// C-ABI entry points declared in include/ktb200.h.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#define KTB_IQ_CODEBOOKS
#include "gemv_bulk.cuh"
#include "dense_bulk.cuh"
#include "rawint4.cuh"
#include "iq.cuh"
#include "handles.cuh"

namespace ktb {

// ------------------------------------------------------------------------------------------
// Q6_K "8-row SoA" re-layout, in place.  For every group of 8 consecutive rows (nb blocks each):
//   raw : row r, block b at (r*nb + b)*210 : {ql[128] qh[64] scales[16] d[2]}
//   soa : [ql: r][b][128] | [qh: r][b][64] | [scales: r][b][16] | [d: r][b][2]
// Same byte count; every slice a lane loads becomes 16-byte aligned (210-byte raw blocks are only
// 2-byte aligned, which would force 16-bit loads).  One CTA per 8-row group, staged through smem.
__global__ void __launch_bounds__(256) repack_q6k_kernel(uint8_t* w, long n_groups, int nb) {
    extern __shared__ __align__(16) uint8_t smem[];
    const long gbytes = 8L * SZ_Q6_K * nb;  // multiple of 16
    for (long g = blockIdx.x; g < n_groups; g += gridDim.x) {
        uint8_t* base = w + g * gbytes;
        for (long i = threadIdx.x; i < gbytes / 16; i += blockDim.x)
            reinterpret_cast<uint4*>(smem)[i] = reinterpret_cast<const uint4*>(base)[i];
        __syncthreads();
        const uint16_t* src = reinterpret_cast<const uint16_t*>(smem);
        uint16_t* dst = reinterpret_cast<uint16_t*>(base);
        const long s_qh = 1024L * nb, s_sc = 1536L * nb, s_d = 1664L * nb;
        for (long i = threadIdx.x; i < gbytes / 2; i += blockDim.x) {
            const long off = 2 * i;
            long r, b, x, sect;
            if (off < s_qh) {
                r = off / (128L * nb); b = (off % (128L * nb)) / 128; x = off % 128; sect = 0;
            } else if (off < s_sc) {
                const long o = off - s_qh;
                r = o / (64L * nb); b = (o % (64L * nb)) / 64; x = o % 64; sect = 128;
            } else if (off < s_d) {
                const long o = off - s_sc;
                r = o / (16L * nb); b = (o % (16L * nb)) / 16; x = o % 16; sect = 192;
            } else {
                const long o = off - s_d;
                r = o / (2L * nb); b = (o % (2L * nb)) / 2; x = 0; sect = 208;
            }
            dst[i] = src[((r * nb + b) * SZ_Q6_K + sect + x) / 2];
        }
        __syncthreads();
    }
}

static int repack_q6k(void* w, long rows_total, int ncols, int device, cudaStream_t stream) {
    const int nb = ncols / QK_K;
    const long n_groups = rows_total / 8;
    const size_t smem = (size_t)8 * SZ_Q6_K * nb;
    if (smem > 200 * 1024) {
        set_error("Q6_K repack: row too long (%d cols)", ncols);
        return KTB200_EINVAL;
    }
    KTB_CUDA_CHECK(cudaFuncSetAttribute(repack_q6k_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    long grid = n_groups < (long)num_sms(device) * 8 ? n_groups : (long)num_sms(device) * 8;
    if (grid < 1) grid = 1;
    repack_q6k_kernel<<<(unsigned)grid, 256, smem, stream>>>(reinterpret_cast<uint8_t*>(w), n_groups, nb);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// ------------------------------------------------------------------------------------------
// Q6_K "4-row chunk-major tile" re-layout, in place (consumed by reduce_bulk_kernel<BulkQ6K4T>, gemv_bulk.cuh).
// Item = 4 consecutive rows x nb blocks (f = rw*nb + blk is also the raw block index inside the item):
//   raw : block f at f*210 : {ql[128] qh[64] scales[16] d[2]}
//   t4  : [ql: c=0..7][f][16] | [qh: c=0..3][f][16] | [scales: f][16] | [d: f][2]
// Same bytes; the item is one contiguous, 16-byte aligned range (nb even) = one bulk copy, and consecutive
// lanes read consecutive 16-byte words of a chunk.
__global__ void __launch_bounds__(256) repack_q6k4t_kernel(uint8_t* w, long n_items, int nb) {
    extern __shared__ __align__(16) uint8_t smem[];
    const long nrb = 4L * nb, ibytes = nrb * SZ_Q6_K;  // multiple of 16 (nb even)
    for (long it = blockIdx.x; it < n_items; it += gridDim.x) {
        uint8_t* base = w + it * ibytes;
        for (long i = threadIdx.x; i < ibytes / 16; i += blockDim.x)
            reinterpret_cast<uint4*>(smem)[i] = reinterpret_cast<const uint4*>(base)[i];
        __syncthreads();
        const uint16_t* src = reinterpret_cast<const uint16_t*>(smem);
        uint16_t* dst = reinterpret_cast<uint16_t*>(base);
        const long s_qh = nrb * 128, s_sc = nrb * 192, s_d = nrb * 208;
        for (long i = threadIdx.x; i < ibytes / 2; i += blockDim.x) {
            const long off = 2 * i;
            long f, sect, x;
            if (off < s_qh) {
                const long c = off / (nrb * 16), o = off % (nrb * 16);
                f = o / 16; x = c * 16 + o % 16; sect = 0;
            } else if (off < s_sc) {
                const long o2 = off - s_qh, c = o2 / (nrb * 16), o = o2 % (nrb * 16);
                f = o / 16; x = c * 16 + o % 16; sect = 128;
            } else if (off < s_d) {
                const long o = off - s_sc;
                f = o / 16; x = o % 16; sect = 192;
            } else {
                f = (off - s_d) / 2; x = 0; sect = 208;
            }
            dst[i] = src[(f * SZ_Q6_K + sect + x) / 2];
        }
        __syncthreads();
    }
}

static int repack_q6k4t(void* w, long rows_total, int ncols, int device, cudaStream_t stream) {
    const int nb = ncols / QK_K;
    const long n_items = rows_total / 4;
    const size_t smem = (size_t)4 * SZ_Q6_K * nb;
    if (smem > 200 * 1024 || nb % 2 || rows_total % 4) {
        set_error("Q6_K tile repack: unsupported shape (%ld rows x %d cols)", rows_total, ncols);
        return KTB200_EINVAL;
    }
    KTB_CUDA_CHECK(cudaFuncSetAttribute(repack_q6k4t_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    long grid = n_items < (long)num_sms(device) * 8 ? n_items : (long)num_sms(device) * 8;
    if (grid < 1) grid = 1;
    repack_q6k4t_kernel<<<(unsigned)grid, 256, smem, stream>>>(reinterpret_cast<uint8_t*>(w), n_items, nb);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// ------------------------------------------------------------------------------------------
// kernel dispatch
template <typename K>
static int set_smem_attr(K kernel, size_t smem) {
    if (smem > 48 * 1024) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    return KTB200_OK;
}

// Tuning knobs (read once): KTB200_MINB = CTAs per SM the main kernels are compiled/launched for (2 or 3),
// KTB200_NB = steps per load batch for the long-row gate/up kernel (2 or 4).
static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}
static int cfg_minb() { static int v = env_int("KTB200_MINB", 2); return v == 3 ? 3 : 2; }
static int cfg_pipe() { static int v = env_int("KTB200_PIPE", 2); return v; }   // 0 off, 1 chunk-per-lane, 2 block-per-lane
static int cfg_nb() { static int v = env_int("KTB200_NB", 2); return v == 4 ? 4 : 2; }
// bulk-copy generation (gemv_bulk.cuh): KTB200_BULK=0 disables it, *_SLOTS_* = ring depth, KTB200_BULK_WARPS caps the CTA
static int cfg_bulk() { static int v = env_int("KTB200_BULK", 1); return v; }
static int cfg_bulk_slots_up() { static int v = env_int("KTB200_BULK_SLOTS_UP", 3); return v == 2 ? 2 : (v == 4 ? 4 : 3); }
static int cfg_bulk_slots_down() { static int v = env_int("KTB200_BULK_SLOTS_DOWN", 2); return v == 3 ? 3 : 2; }
static int cfg_bulk_warps() { static int v = env_int("KTB200_BULK_WARPS", kBulkMaxWarps); return v < 1 ? 1 : (v > kBulkMaxWarps ? kBulkMaxWarps : v); }
constexpr size_t kSmemCap = 232448 - 512;   // 227 KB opt-in limit minus the kernels' static shared variables

template <class Fmt, bool PAIR>
static int launch_rows_fmt(const RowsParams& p, int T, int device, cudaStream_t stream, bool tunable) {
    const int nblk = p.ncols / QK_K;
    const int nsteps = (nblk + Fmt::kBlocksPerStep - 1) / Fmt::kBlocksPerStep;
    const size_t smem = (size_t)p.ncols + (size_t)nblk * 4 + (size_t)p.ncols / 8;
    const int minb = tunable ? cfg_minb() : 2;
    int gx = (minb * num_sms(device) + T - 1) / T;
    const long total = (long)(p.slots + (p.x0 ? 1 : 0)) * p.rows;
    if (total >= (1L << 31) / 2) { set_error("rows kernel: slots x rows too large"); return KTB200_EINVAL; }
    if (gx > total) gx = (int)total;
    if (gx < 1) gx = 1;
    dim3 grid(gx, T);
#define KTB_ROWS(RW, NB, MINB)                                                             \
    do {                                                                                   \
        int rc = set_smem_attr(rows_kernel<Fmt, PAIR, RW, NB, MINB>, smem);                \
        if (rc) return rc;                                                                 \
        rows_kernel<Fmt, PAIR, RW, NB, MINB><<<grid, kGemvThreads, smem, stream>>>(p);     \
    } while (0)
    if (nsteps >= 4) {
        if (tunable && minb == 3) KTB_ROWS(1, 2, 3);
        else if (tunable && cfg_nb() == 2) KTB_ROWS(1, 2, 2);
        else KTB_ROWS(1, 4, 2);
    } else if (nsteps >= 2) KTB_ROWS(2, 2, 2);
    else KTB_ROWS(4, 1, 2);
#undef KTB_ROWS
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// cp.async-pipelined variant (gemv_pipe.cuh): one CTA per SM, a private 2-slot ring per warp.
// Returns 1 when the shape does not suit it (caller falls back to rows_kernel).
template <class Fmt, bool PAIR>
static int launch_rows_pipe(const RowsParams& p, int T, int device, cudaStream_t stream) {
    if (!cfg_pipe()) return 1;
    const int nblk = p.ncols / QK_K;
    const int row_bytes = nblk * Fmt::kBlockBytes;
    const int slot = row_bytes * (PAIR ? 2 : 1);
    const int act = (p.ncols + ((nblk * 4 + 15) & ~15) + p.ncols / 8 + 15) & ~15;
    if (slot < 4096) return 1;                          // short rows: the register-staged kernel batches better
    int warps = 0;
    for (int w : {12, 8}) if ((size_t)act + (size_t)w * 2 * slot <= 220 * 1024) { warps = w; break; }
    if (!warps) return 1;
    const size_t smem = (size_t)act + (size_t)warps * 2 * slot;
    const long total = (long)(p.slots + (p.x0 ? 1 : 0)) * p.rows;
    if (total >= (1L << 30)) return 1;
    int gx = (num_sms(device) + T - 1) / T;
    if (gx > total) gx = (int)total;
    if (gx < 1) gx = 1;
    dim3 grid(gx, T);
    if (warps == 12) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(rows_pipe_kernel<Fmt, PAIR, 12>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rows_pipe_kernel<Fmt, PAIR, 12><<<grid, 12 * 32, smem, stream>>>(p, act, slot);
    } else {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(rows_pipe_kernel<Fmt, PAIR, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rows_pipe_kernel<Fmt, PAIR, 8><<<grid, 8 * 32, smem, stream>>>(p, act, slot);
    }
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// Q4_K rows through the bulk-copy ring (rows_bulk_q4k_kernel).  Returns 1 when the shape does not suit it.
template <bool PAIR>
static int launch_rows_bulk_q4k(const RowsParams& p, int T, int device, cudaStream_t stream) {
    if (!cfg_bulk()) return 1;
    const int nblk = p.ncols / QK_K;
    const int row_bytes = nblk * SZ_Q4_K;
    if (nblk < 16) return 1;                             // needs >= 16 blocks per row to keep most lanes busy
    const int nslots = p.slots + (p.x0 ? 1 : 0);
    const long total = (long)nslots * p.rows;
    if (total >= (1L << 26) || nslots > 200) return 1;
    const int act_tok = (nblk * kActBlkStride + nblk * 16 + nblk * 4 + 15) & ~15;
    const int S = cfg_bulk_slots_up();
    // tokens per chunk: as many (<= 8) as fit next to 12 rings; then as many warps as fit
    int tc = T < 8 ? T : 8;
    while (tc > 1 && (size_t)tc * (act_tok + nslots * 4) + 64 + (size_t)12 * S * (row_bytes + 8) > kSmemCap) tc--;
    const size_t head = (((size_t)tc * act_tok + (size_t)tc * nslots * 4 + 15) & ~(size_t)15);
    if (head + 64 >= kSmemCap) return 1;
    int W = (int)((kSmemCap - head - 16) / ((size_t)S * (row_bytes + 8)));
    if (W > cfg_bulk_warps()) W = cfg_bulk_warps();
    if (W < 4) return 1;
    const size_t smem = head + (((size_t)W * S * 8 + 15) & ~(size_t)15) + (size_t)W * S * row_bytes;
    int gx = num_sms(device);            // one CTA per SM walks all T tokens
    if (gx > total) gx = (int)total;
    if (gx < 1) gx = 1;
#define KTB_BULK_ROWS(SL)                                                                                              \
    do {                                                                                                               \
        KTB_CUDA_CHECK(cudaFuncSetAttribute(rows_bulk_q4k_kernel<PAIR, SL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        rows_bulk_q4k_kernel<PAIR, SL><<<gx, W * 32, smem, stream>>>(p, act_tok, tc);                                  \
    } while (0)
    if (S == 2) KTB_BULK_ROWS(2); else if (S == 4) KTB_BULK_ROWS(4); else KTB_BULK_ROWS(3);
#undef KTB_BULK_ROWS
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// Dense Q4_K linear on the segment ring (dense_bulk.cuh).  Returns 1 when the shape does not suit it.
static int launch_dense_q4k(const RowsParams& p, int T, int device, cudaStream_t stream) {
    static const int on = env_int("KTB200_DENSE_BULK", 1);
    if (!on || p.ids || p.slots != 1 || p.x0 || !p.out_hidden || p.out_f32 || T > kDenseMaxTokens) return 1;
    const int nblk = p.ncols / QK_K;
    DenseParams d{};
    d.w = reinterpret_cast<const uint8_t*>(p.w0); d.x = p.x; d.out = p.out_hidden; d.bias = p.bias; d.bsz = p.bsz;
    d.rows = p.rows; d.ncols = p.ncols; d.T = T; d.hidden_type = p.hidden_type;
    if (nblk <= 16) { d.R = 32 / nblk; d.G = 1; d.segb = d.R * nblk; }
    else if (nblk <= 32) { d.R = 1; d.G = 1; d.segb = nblk; }
    else { d.R = 1; d.G = (nblk + 31) / 32; if (nblk % d.G) return 1; d.segb = nblk / d.G; }
    d.act_tok = (nblk * kActBlkStride + nblk * 16 + nblk * 4 + 15) & ~15;
    constexpr int SL = 4;
    const size_t head = (((size_t)T * d.act_tok + 15) & ~(size_t)15);
    const size_t seg = (size_t)d.segb * SZ_Q4_K;
    if (head + 64 >= kSmemCap) return 1;
    int W = (int)((kSmemCap - head - 16) / (SL * (seg + 8)));
    if (W > kDenseWarps) W = kDenseWarps;
    if (W < 4) return 1;
    const size_t smem = head + (((size_t)W * SL * 8 + 15) & ~(size_t)15) + (size_t)W * SL * seg;
    const int nunits = (p.rows + d.R - 1) / d.R;
    int gx = num_sms(device);
    if (gx > nunits) gx = nunits;
    static size_t limit[64] = {};
    if (limit[device & 63] < smem) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(dense_q4k_kernel<SL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        limit[device & 63] = smem;
    }
    KTB_CUDA_CHECK(launch_pdl(dense_q4k_kernel<SL>, dim3(gx), dim3(W * 32), smem, stream, d));
    count_launch();
    return KTB200_OK;
}

// RAWINT4 gate/up pairs (rows_bulk_i4_kernel): the only kernel for the format, so a shape it cannot take is an error.
// Ring of 2 slots per warp (one (gate row | up row) pair in flight while one is computed); tokens per chunk: as many
// (<= 8) as leave room for >= 8 warps.
static int launch_rows_i4(const RowsParams& p, int T, int device, cudaStream_t stream) {
    constexpr int S = 2;
    const int nblk = p.ncols / QK_K;
    const size_t slot = (size_t)2 * nblk * SZ_RAWINT4;
    const size_t act_tok = (size_t)nblk * kI4ActStride;
    const long total = (long)p.slots * p.rows;
    if (p.x0 || p.shared_token >= 0 || p.slots > 200 || total >= (1L << 26)) { set_error("RAWINT4 gate/up: unsupported launch"); return KTB200_EINVAL; }
    auto head = [&](int tc) { return ((size_t)tc * act_tok + (size_t)tc * p.slots * 4 + 15) & ~(size_t)15; };
    int tc = T < kI4MaxChunkTokens ? T : kI4MaxChunkTokens;
    while (tc > 1 && head(tc) + 64 + (size_t)8 * S * (slot + 8) > kSmemCap) tc--;
    if (head(tc) + 64 >= kSmemCap) { set_error("RAWINT4 gate/up: hidden_size %d does not fit shared memory", p.ncols); return KTB200_EINVAL; }
    int W = (int)((kSmemCap - head(tc) - 16) / (S * (slot + 8)));
    if (W > cfg_bulk_warps()) W = cfg_bulk_warps();
    if (W < 1) { set_error("RAWINT4 gate/up: hidden_size %d does not fit shared memory", p.ncols); return KTB200_EINVAL; }
    const size_t smem = head(tc) + (((size_t)W * S * 8 + 15) & ~(size_t)15) + (size_t)W * S * slot;
    int gx = num_sms(device);
    if (gx > total) gx = (int)total;
    if (gx < 1) gx = 1;
    KTB_CUDA_CHECK(cudaFuncSetAttribute(rows_bulk_i4_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rows_bulk_i4_kernel<S><<<gx, W * 32, smem, stream>>>(p, tc);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// IQ1_S / IQ2_XXS gate/up pairs through the bulk-copy ring (rows_bulk_iq_kernel, iq.cuh): 2-row units, 2 slots per warp,
// tokens per chunk as many (<= 8) as leave room for >= 8 warps.  Returns 1 when the launch does not suit it (gate and up
// of different types, rows not 16-byte aligned in pairs, a shared-expert slot): the generic kernels take it then.
template <class Fmt>
static int launch_rows_bulk_iq(const RowsParams& p, int T, int device, cudaStream_t stream) {
    constexpr int S = 2;
    if (!cfg_bulk()) return 1;
    const int nblk = p.ncols / QK_K;
    if (p.type0 != Fmt::kType || p.type1 != Fmt::kType || p.x0 || !p.ids || nblk % 4 || p.rows % 2 || p.slots > 200) return 1;
    const long total = (long)p.slots * (p.rows / 2);
    if (total >= (1L << 26)) return 1;
    const size_t slot = (size_t)4 * nblk * Fmt::kBlockBytes;
    const int act_tok = (nblk * kActBlkStride + nblk * 16 + nblk * 4 + 15) & ~15;
    const size_t cap = kSmemCap - Fmt::kTableBytes;
    auto head = [&](int tc) { return ((size_t)tc * act_tok + (size_t)tc * p.slots * 4 + 15) & ~(size_t)15; };
    int tc = T < 8 ? T : 8;
    while (tc > 1 && head(tc) + 64 + (size_t)8 * S * (slot + 8) > cap) tc--;
    if (head(tc) + 64 >= cap) return 1;
    int W = (int)((cap - head(tc) - 16) / (S * (slot + 8)));
    if (W > kIqMaxWarps) W = kIqMaxWarps;
    if (W > cfg_bulk_warps()) W = cfg_bulk_warps();
    if (W < 4) return 1;
    const size_t smem = head(tc) + (((size_t)W * S * 8 + 15) & ~(size_t)15) + (size_t)W * S * slot;
    int gx = num_sms(device);
    if (gx > total) gx = (int)total;
    if (gx < 1) gx = 1;
    KTB_CUDA_CHECK(cudaFuncSetAttribute(rows_bulk_iq_kernel<Fmt, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rows_bulk_iq_kernel<Fmt, S><<<gx, W * 32, smem, stream>>>(p, act_tok, tc);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

template <bool PAIR>
static int launch_rows(FmtId f, const RowsParams& p_in, int T, int device, cudaStream_t stream) {
    RowsParams p = p_in;
    p.ntokens = T;
    if (f == FMT_RAWINT4) {
        if (!PAIR) { set_error("RAWINT4: routed experts only"); return KTB200_EINVAL; }
        return launch_rows_i4(p, T, device, stream);
    }
    if (PAIR && f == FMT_GENK && is_iquant(p.type0)) {
        const int rci = p.type0 == KTB200_TYPE_IQ1_S ? launch_rows_bulk_iq<BulkIQ1S>(p, T, device, stream)
                                                     : launch_rows_bulk_iq<BulkIQ2XXS>(p, T, device, stream);
        if (rci != 1) return rci;
    }
    if (!PAIR && f == FMT_Q4K) {
        const int rcd = launch_dense_q4k(p, T, device, stream);
        if (rcd != 1) return rcd;
    }
    if (f == FMT_Q4K) {
        const int rcb = launch_rows_bulk_q4k<PAIR>(p, T, device, stream);
        if (rcb != 1) return rcb;
    }
    if (p.x0 && p.shared_token >= 0) { set_error("per-token shared slot: only the bulk-copy kernels implement it"); return KTB200_EINVAL; }
    if (f == FMT_Q4K || f == FMT_Q5K) {
        const int rc = (f == FMT_Q4K) ? launch_rows_pipe<FmtQ4K32, PAIR>(p, T, device, stream) : launch_rows_pipe<FmtQ5K, PAIR>(p, T, device, stream);
        if (rc != 1) return rc;
    }
    switch (f) {
        case FMT_Q4K: return launch_rows_fmt<FmtQ4K, PAIR>(p, T, device, stream, true);
        case FMT_Q5K: return launch_rows_fmt<FmtQ5K, PAIR>(p, T, device, stream, false);
        case FMT_Q6K8: return launch_rows_fmt<FmtQ6K8, PAIR>(p, T, device, stream, false);
        case FMT_GENK: return launch_rows_fmt<FmtGenK, PAIR>(p, T, device, stream, false);
        default: set_error("unsupported weight type"); return KTB200_EINVAL;
    }
}

template <class Fmt, int NBMAX>
static int launch_reduce_fmt(const ReduceParams& p, int T, int device, cudaStream_t stream, bool tunable) {
    const int nblk = p.ncols / QK_K;
    const int nsteps = (nblk + Fmt::kBlocksPerStep - 1) / Fmt::kBlocksPerStep;
    const int minb = tunable ? cfg_minb() : 2;
    const int ns = p.slots + (p.xw ? 1 : 0);
    int gx = (minb * num_sms(device) + T - 1) / T;
    if (gx > p.rows) gx = p.rows;
    if (gx < 1) gx = 1;
    const int nrows_max = (p.rows + gx - 1) / gx + 1;
    const size_t per_slot = (size_t)p.ncols + (size_t)nblk * 4 + (size_t)p.ncols / 8;
    const size_t smem = per_slot * ns + (size_t)nrows_max * ns * 4;
    if (smem > 220 * 1024) {
        set_error("reduce kernel: k=%d x ncols=%d does not fit shared memory", ns, p.ncols);
        return KTB200_EINVAL;
    }
    dim3 grid(gx, T);
#define KTB_RED(NB, MINB)                                                                  \
    do {                                                                                   \
        int rc = set_smem_attr(reduce_kernel<Fmt, NB, MINB>, smem);                        \
        if (rc) return rc;                                                                 \
        reduce_kernel<Fmt, NB, MINB><<<grid, kGemvThreads, smem, stream>>>(p);             \
    } while (0)
    if (NBMAX >= 2 && nsteps >= 2) {
        if (minb == 3) KTB_RED((NBMAX >= 2 ? 2 : 1), 3); else KTB_RED((NBMAX >= 2 ? 2 : 1), 2);
    } else {
        if (minb == 3) KTB_RED(1, 3); else KTB_RED(1, 2);
    }
#undef KTB_RED
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// cp.async-pipelined Q6_K (SoA) reduce: returns 1 when the shape does not suit it
static int launch_reduce_pipe_q6k8(const ReduceParams& p, int T, int device, cudaStream_t stream) {
    if (!cfg_pipe()) return 1;
    const int nb = p.ncols / QK_K;
    if (p.rows % 4 || nb % 2) return 1;
    const int ns = p.slots + (p.xw ? 1 : 0);
    const int slot = 840 * nb;     // 4 rows x 210 nb
    if (slot < 4096) return 1;
    const int quads = p.rows / 4;
    int gx = (num_sms(device) + T - 1) / T;
    if (gx > quads) gx = quads;
    if (gx < 1) gx = 1;
    const int nrows_max = ((quads + gx - 1) / gx + 1) * 4;
    size_t base = (size_t)ns * p.ncols + (size_t)ns * nb * 4 + (size_t)ns * (p.ncols / 16) * 2 + (size_t)nrows_max * ns * 4 + 16;
    static const int want_slots = env_int("KTB200_PIPE_SLOTS", 2);
    dim3 grid(gx, T);
    if (want_slots != 2 && base + (size_t)24 * slot <= 220 * 1024) {
        const size_t smem = base + (size_t)24 * slot;
        KTB_CUDA_CHECK(cudaFuncSetAttribute(reduce_pipe_q6k8_kernel<24, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        reduce_pipe_q6k8_kernel<24, 1><<<grid, 24 * 32, smem, stream>>>(p, slot);
    } else if (base + (size_t)12 * 2 * slot <= 220 * 1024) {
        const size_t smem = base + (size_t)12 * 2 * slot;
        KTB_CUDA_CHECK(cudaFuncSetAttribute(reduce_pipe_q6k8_kernel<12, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        reduce_pipe_q6k8_kernel<12, 2><<<grid, 12 * 32, smem, stream>>>(p, slot);
    } else {
        return 1;
    }
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// Shared-memory plan of reduce_bulk_kernel<Fmt, S> for `pcap` staged (token, slot) pairs: returns the warp count
// (0 = does not fit)
template <class Fmt>
static int reduce_bulk_plan(int rows, int ncols, int pcap, int S, int device, int* gx_out, int* nrows_max_out, size_t* smem_out) {
    const int nb = ncols / QK_K;
    if (rows % 4 || nb < 1 || pcap > 200) return 0;
    const size_t item = (size_t)4 * nb * Fmt::kBlockBytes;
    if (item % 16) return 0;
    const int quads = rows / 4;
    int gx = num_sms(device);
    if (gx > quads) gx = quads;
    if (gx < 1) gx = 1;
    const int nrows_max = ((quads + gx - 1) / gx) * 4;
    size_t base = (size_t)pcap * nb * (kActBlkStride + 2 * Fmt::kBs + 4) + (size_t)nrows_max * pcap * 4 + (size_t)pcap * 4;
    base = (base + 15) & ~(size_t)15;
    const size_t cap = kSmemCap - Fmt::kTableBytes;
    if (base + 16 >= cap) return 0;
    int W = (int)((cap - base - 16) / ((size_t)S * (item + 8)));
    if (W > cfg_bulk_warps()) W = cfg_bulk_warps();
    if (W > kBulkMaxWarpsDown) W = kBulkMaxWarpsDown;
    if (W < 2) return 0;
    if (gx_out) *gx_out = gx;
    if (nrows_max_out) *nrows_max_out = nrows_max;
    if (smem_out) *smem_out = base + (((size_t)W * S * 8 + 15) & ~(size_t)15) + (size_t)W * S * item;
    return W;
}

// Down projection through the bulk-copy ring.  Returns 1 when the shape does not suit it.
template <class Fmt>
static int launch_reduce_bulk(const ReduceParams& p, int T, int device, cudaStream_t stream) {
    if (!cfg_bulk()) return 1;
    const int ns = p.slots + (p.xw ? 1 : 0);
    const int S = cfg_bulk_slots_down();
    // pair capacity of a token chunk: one token's worth at least; up to 2 tokens' worth (<= 18) when several tokens
    // share the launch and >= 10 warps still fit
    int pcap = ns;
    if (T > 1) {
        int want = 2 * ns < 18 ? 2 * ns : (ns > 18 ? ns : 18);
        if ((long)T * ns < want) want = T * ns;
        while (want > ns && reduce_bulk_plan<Fmt>(p.rows, p.ncols, want, S, device, nullptr, nullptr, nullptr) < 10) want--;
        pcap = want;
    }
    int gx = 0, nrows_max = 0;
    size_t smem = 0;
    const int W = reduce_bulk_plan<Fmt>(p.rows, p.ncols, pcap, S, device, &gx, &nrows_max, &smem);
    if (!W) return 1;
    if (S == 3) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(reduce_bulk_kernel<Fmt, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        reduce_bulk_kernel<Fmt, 3><<<gx, W * 32, smem, stream>>>(p, nrows_max, pcap);
    } else {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(reduce_bulk_kernel<Fmt, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        reduce_bulk_kernel<Fmt, 2><<<gx, W * 32, smem, stream>>>(p, nrows_max, pcap);
    }
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// Load-time decision: can a Q6_K down tensor [rows][ncols] take the T4 tile layout (and therefore ONLY the bulk
// kernel) for up to ns_max slots per token?
static bool q6k4t_eligible(int rows, int ncols, int ns_max, int device) {
    if (!cfg_bulk()) return false;
    const int nb = ncols / QK_K;
    if (nb % 2 || rows % 4) return false;
    return reduce_bulk_plan<BulkQ6K4T>(rows, ncols, ns_max, 3, device, nullptr, nullptr, nullptr) >= 4;
}

// Shared-memory plan of reduce_bulk_i4_kernel<S> for `pcap` staged pairs: returns the warp count (0 = does not fit)
static int reduce_i4_plan(int rows, int ncols, int pcap, int S, int device, int* gx_out, int* nrows_max_out, size_t* smem_out) {
    const int nb = ncols / QK_K;
    if (rows % 4 || nb < 1 || pcap > 200) return 0;
    const size_t item = (size_t)4 * nb * SZ_RAWINT4;
    const int quads = rows / 4;
    int gx = num_sms(device);
    if (gx > quads) gx = quads;
    if (gx < 1) gx = 1;
    const int nrows_max = ((quads + gx - 1) / gx) * 4;
    size_t base = (size_t)pcap * nb * kI4ActStride + (size_t)nrows_max * pcap * 4 + (size_t)pcap * 4;
    base = (base + 15) & ~(size_t)15;
    if (base + 16 >= kSmemCap) return 0;
    int W = (int)((kSmemCap - base - 16) / ((size_t)S * (item + 8)));
    if (W > cfg_bulk_warps()) W = cfg_bulk_warps();
    if (W > kBulkMaxWarpsDown) W = kBulkMaxWarpsDown;
    if (W < 1) return 0;
    if (gx_out) *gx_out = gx;
    if (nrows_max_out) *nrows_max_out = nrows_max;
    if (smem_out) *smem_out = base + (((size_t)W * S * 8 + 15) & ~(size_t)15) + (size_t)W * S * item;
    return W;
}

// RAWINT4 down projection (reduce_bulk_i4_kernel): pair capacity of a token chunk as in launch_reduce_bulk.
static int launch_reduce_i4(const ReduceParams& p, int T, int device, cudaStream_t stream) {
    constexpr int S = 2;
    if (p.xw) { set_error("RAWINT4 down: the shared expert cannot ride in the routed launch"); return KTB200_EINVAL; }
    const int ns = p.slots;
    int pcap = ns;
    if (T > 1) {
        int want = 2 * ns < 18 ? 2 * ns : (ns > 18 ? ns : 18);
        if ((long)T * ns < want) want = T * ns;
        while (want > ns && reduce_i4_plan(p.rows, p.ncols, want, S, device, nullptr, nullptr, nullptr) < 10) want--;
        pcap = want;
    }
    int gx = 0, nrows_max = 0;
    size_t smem = 0;
    const int W = reduce_i4_plan(p.rows, p.ncols, pcap, S, device, &gx, &nrows_max, &smem);
    if (!W) { set_error("RAWINT4 down: k=%d x intermediate_size=%d does not fit shared memory", ns, p.ncols); return KTB200_EINVAL; }
    KTB_CUDA_CHECK(cudaFuncSetAttribute(reduce_bulk_i4_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    reduce_bulk_i4_kernel<S><<<gx, W * 32, smem, stream>>>(p, nrows_max, pcap);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

static int launch_reduce(FmtId f, const ReduceParams& p_in, int T, int device, cudaStream_t stream) {
    ReduceParams p = p_in;
    p.ntokens = T;
    if (f == FMT_RAWINT4) return launch_reduce_i4(p, T, device, stream);
    if (f == FMT_Q6K4T) {
        const int rc = launch_reduce_bulk<BulkQ6K4T>(p, T, device, stream);
        if (rc == 1) { set_error("Q6_K tile layout: k=%d x ncols=%d does not fit the bulk kernel", p.slots, p.ncols); return KTB200_EINVAL; }
        return rc;
    }
    if (f == FMT_Q4K) {
        const int rc = launch_reduce_bulk<BulkQ4K>(p, T, device, stream);
        if (rc != 1) return rc;
    }
    if (f == FMT_GENK && is_iquant(p.type) && !p.xw) {   // IQ down items (iq.cuh); otherwise the generic kernel
        const int rc = p.type == KTB200_TYPE_IQ1_S ? launch_reduce_bulk<BulkIQ1S>(p, T, device, stream)
                                                   : launch_reduce_bulk<BulkIQ2XXS>(p, T, device, stream);
        if (rc != 1) return rc;
    }
    if (p.xw && (p.shared_token >= 0 || p.xw_out)) { set_error("per-token shared slot: only the bulk-copy kernels implement it"); return KTB200_EINVAL; }
    if (f == FMT_Q6K8) {
        const int rc = launch_reduce_pipe_q6k8(p, T, device, stream);
        if (rc != 1) return rc;
    }
    switch (f) {
        case FMT_Q4K: return launch_reduce_fmt<FmtQ4K, 2>(p, T, device, stream, true);
        case FMT_Q5K: return launch_reduce_fmt<FmtQ5K, 1>(p, T, device, stream, false);
        case FMT_Q6K8: return launch_reduce_fmt<FmtQ6K8, 1>(p, T, device, stream, true);
        case FMT_GENK: return launch_reduce_fmt<FmtGenK, 1>(p, T, device, stream, false);
        default: set_error("unsupported weight type"); return KTB200_EINVAL;
    }
}

static bool weight_type_ok(int t) { return is_kquant(t); }
// routed experts also take the codebook i-quants (generic per-pair kernels; IQ down-projection items)
static bool expert_type_ok(int t) { return is_kquant(t) || is_iquant(t); }

// quantize API kernel: one warp per 256-block, packed block_q8_K output (292 B)
__global__ void __launch_bounds__(256) quantize_q8k_kernel(const void* x, int hidden_type, long n_blocks, uint8_t* out) {
    const int lane = threadIdx.x & 31;
    const long b = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= n_blocks) return;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = load_hidden(x, b * QK_K + lane * 8 + i, hidden_type);
    uint8_t* blk = out + b * SZ_Q8_K;
    warp_quantize_q8k_block(v, lane, reinterpret_cast<uint32_t*>(blk + 4), reinterpret_cast<float*>(blk),
                            reinterpret_cast<int16_t*>(blk + 4 + QK_K));
}
__global__ void __launch_bounds__(256) quantize_q8_0_kernel(const void* x, int hidden_type, long n_blocks, uint8_t* out) {
    const int lane = threadIdx.x & 31;
    const long b = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= n_blocks) return;
    float d;
    uint8_t* blk = out + b * SZ_Q8_0;
    warp_quantize_q8_0_block(load_hidden(x, b * 32 + lane, hidden_type), lane, reinterpret_cast<int8_t*>(blk + 2), &d,
                             reinterpret_cast<uint16_t*>(blk));
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb200_moe_create(const ktb200_moe_config* c, int device, ktb200_moe** out) {
    if (!c || !out) { set_error("null argument"); return KTB200_EINVAL; }
    if (c->expert_num <= 0 || c->routed_expert_num <= 0 || c->hidden_size <= 0 || c->intermediate_size <= 0 ||
        c->group_max_len <= 0) { set_error("MOEConfig: non-positive dimension"); return KTB200_EINVAL; }
    const int n_i4 = is_rawint4(c->gate_type) + is_rawint4(c->up_type) + is_rawint4(c->down_type);
    if (n_i4 != 0 && n_i4 != 3) {
        set_error("MOEConfig: RAWINT4_G32 must be the type of all three tensors (gate %d up %d down %d)", c->gate_type, c->up_type, c->down_type);
        return KTB200_EINVAL;
    }
    if (!n_i4 && (!expert_type_ok(c->gate_type) || !expert_type_ok(c->up_type) || !expert_type_ok(c->down_type))) {
        set_error("MOEConfig: unsupported ggml weight type (gate %d up %d down %d)", c->gate_type, c->up_type, c->down_type);
        return KTB200_EINVAL;
    }
    if (!is_hidden_type(c->hidden_type)) { set_error("MOEConfig: hidden_type %d must be F32/F16/BF16", c->hidden_type); return KTB200_EINVAL; }
    if (c->hidden_size % QK_K || c->intermediate_size % QK_K) {
        set_error("MOEConfig: hidden_size %d and intermediate_size %d must be multiples of 256 for K-quant tensors",
                  c->hidden_size, c->intermediate_size);
        return KTB200_EINVAL;
    }
    if (!c->gate_proj || !c->up_proj || !c->down_proj) { set_error("MOEConfig: null weight pointer"); return KTB200_EINVAL; }
    DeviceGuard g(device);
    if (!g.ok) { set_error("cudaSetDevice(%d) failed", device); return KTB200_ECUDA; }
    ktb200_moe* m = new (std::nothrow) ktb200_moe();
    if (!m) return KTB200_ENOMEM;
    m->cfg = *c;
    m->device = device;
    m->loaded = false;
    m->gu_soa = false;
    m->down_layout = LAYOUT_RAW;
    m->inter = nullptr; m->ids_d = nullptr; m->w_d = nullptr; m->in_d = nullptr; m->out_d = nullptr;
    m->blk_partial = nullptr; m->blk_sync = nullptr; m->blk_flip = 0; m->blk_inter = nullptr; m->blk_stage = nullptr;
    for (int r = 0; r < 3; r++) { m->pf[r] = nullptr; m->pf_bytes[r] = 0; }
    const size_t slots = (size_t)c->group_max_len * c->routed_expert_num;
    const size_t hid = (size_t)c->group_max_len * c->hidden_size * type_size(c->hidden_type);
    // +1 slot per token: the optionally fused shared expert (ktb200_moe_forward_shared)
    cudaError_t e = cudaMalloc(&m->inter, (slots + c->group_max_len) * c->intermediate_size * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&m->ids_d, slots * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMalloc(&m->w_d, slots * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&m->in_d, hid);
    if (e == cudaSuccess) e = cudaMalloc(&m->out_d, hid);
    if (e == cudaSuccess) e = cudaMalloc(&m->blk_partial, (size_t)8 * 8 * 512 * sizeof(float));
    const size_t sync_words = kBlkReadyWord + 2 * blk_ready_words(*c);
    if (e == cudaSuccess) e = cudaMalloc(&m->blk_sync, sync_words * sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMemset(m->blk_sync, 0, sync_words * sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMalloc(&m->blk_inter, blk_ready_words(*c) * QK_K * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(m->blk_inter, 0xff, blk_ready_words(*c) * QK_K * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&m->blk_stage, blk_ready_words(*c) * (QK_K + 32 + 4));
    if (e != cudaSuccess) {
        set_error("cudaMalloc failed: %s", cudaGetErrorString(e));
        ktb200_moe_destroy(m);
        return KTB200_ENOMEM;
    }
    *out = m;
    return KTB200_OK;
}

void ktb200_moe_destroy(ktb200_moe* m) {
    if (!m) return;
    DeviceGuard g(m->device);
    cudaFree(m->inter); cudaFree(m->ids_d); cudaFree(m->w_d); cudaFree(m->in_d); cudaFree(m->out_d);
    cudaFree(m->blk_partial); cudaFree(m->blk_sync); cudaFree(m->blk_inter); cudaFree(m->blk_stage);
    delete m;
}

int ktb200_moe_load_weights(ktb200_moe* m, void* stream) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    if (m->loaded) return KTB200_OK;
    DeviceGuard g(m->device);
    const ktb200_moe_config& c = m->cfg;
    cudaStream_t s = (cudaStream_t)stream;
    if (c.gate_type == KTB200_TYPE_Q6_K && c.up_type == KTB200_TYPE_Q6_K && c.intermediate_size % 8 == 0) {
        int rc = repack_q6k(const_cast<void*>(c.gate_proj), (long)c.expert_num * c.intermediate_size, c.hidden_size, m->device, s);
        if (rc) return rc;
        rc = repack_q6k(const_cast<void*>(c.up_proj), (long)c.expert_num * c.intermediate_size, c.hidden_size, m->device, s);
        if (rc) return rc;
        m->gu_soa = true;
    }
    if (c.down_type == KTB200_TYPE_Q6_K && q6k4t_eligible(c.hidden_size, c.intermediate_size, c.routed_expert_num + 1, m->device)) {
        int rc = repack_q6k4t(const_cast<void*>(c.down_proj), (long)c.expert_num * c.hidden_size, c.intermediate_size, m->device, s);
        if (rc) return rc;
        m->down_layout = LAYOUT_T4;
    } else if (c.down_type == KTB200_TYPE_Q6_K && c.hidden_size % 8 == 0) {
        int rc = repack_q6k(const_cast<void*>(c.down_proj), (long)c.expert_num * c.hidden_size, c.intermediate_size, m->device, s);
        if (rc) return rc;
        m->down_layout = LAYOUT_SOA8;
    }
    m->loaded = true;
    return KTB200_OK;
}

float* ktb200_moe_intermediate(ktb200_moe* m) { return m ? m->inter : nullptr; }

extern "C++" {
namespace ktb {
bool grouped_ok(const ktb200_moe* m, int k);
int moe_forward_grouped(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input, void* output, const int* bsz, cudaStream_t s,
                        int out_type);
void grouped_set_trace(long long* t);
}
}
// qlen from which the per-expert tensor-core GEMMs (grouped.cu) replace the per-pair GEMV kernels: the reference makes the
// same split between MOE::forward_one and MOE::forward_many (moe.cpp:367-377, threshold group_min_len)
void ktb200_debug_grouped(long long* trace_dev) { ktb::grouped_set_trace(trace_dev); }
static int grouped_min_qlen() {
    static const int v = [] { const char* e = getenv("KTB200_GROUPED_MIN"); return e ? atoi(e) : 48; }();
    return v;
}

// out_type: the type of `output` (-1: the handle's hidden_type).  The input rows are always of the hidden type; only the down
// kernels and the grouped combine write `output`, so an F32 out_type yields the unrounded fp32 routed sums.
static int moe_forward_impl(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input,
                            void* output, const int* bsz, cudaStream_t s, cudaEvent_t mid, const ktb200_mlp* sh = nullptr,
                            int shared_token = -1, void* shared_out = nullptr, int out_type = -1) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    if (!m->loaded) { set_error("Not Loaded"); return KTB200_ESTATE; }
    if (qlen <= 0) return KTB200_OK;
    const ktb200_moe_config& c = m->cfg;
    if (k <= 0 || k > c.routed_expert_num) { set_error("forward: k=%d outside (0, routed_expert_num=%d]", k, c.routed_expert_num); return KTB200_EINVAL; }
    if (qlen > c.group_max_len) { set_error("forward: qlen=%d exceeds group_max_len=%d", qlen, c.group_max_len); return KTB200_EINVAL; }
    if (!ids || !weights || !input || !output) { set_error("forward: null pointer"); return KTB200_EINVAL; }
    if (out_type < 0) out_type = c.hidden_type;
    if (out_type != c.hidden_type && sh) { set_error("forward: a shared expert needs the hidden output type"); return KTB200_EINVAL; }
    DeviceGuard g(m->device);

    if (!mid && !shared_out && grouped_min_qlen() > 0 && qlen >= grouped_min_qlen() && grouped_ok(m, k)) {
        int rc = moe_forward_grouped(m, qlen, k, ids, weights, input, output, bsz, s, out_type);
        if (rc || !sh) return rc;
        return ktb200_mlp_forward(const_cast<ktb200_mlp*>(sh), qlen, input, output, 1, bsz, (void*)s);
    }
    FmtId fg = pick_fmt(c.gate_type, m->gu_soa), fu = pick_fmt(c.up_type, m->gu_soa);
    if (fg != fu) fg = fu = FMT_GENK;  // mixed gate/up types: the generic path reads the type per matrix
    RowsParams rp{};
    rp.shared_token = -1;
    rp.w0 = c.gate_proj; rp.w1 = c.up_proj; rp.type0 = c.gate_type; rp.type1 = c.up_type;
    rp.n_experts = c.expert_num; rp.rows = c.intermediate_size; rp.ncols = c.hidden_size; rp.slots = k;
    rp.ids = ids; rp.id_offset = c.expert_id_offset; rp.x = input; rp.hidden_type = c.hidden_type;
    rp.use_silu = c.use_silu; rp.out_f32 = m->inter; rp.out_hidden = nullptr; rp.bias = nullptr; rp.bsz = bsz;
    const FmtId fd = pick_fmt(c.down_type, m->down_layout);
    // the shared expert rides in the same two launches as slot k when its tensors have the routed experts'
    // shapes and layouts (DeepSeek-V3: n_shared_experts = 1, same quant types); otherwise it runs separately
    const bool fuse = sh && sh->loaded && sh->H == c.hidden_size && sh->I == c.intermediate_size && c.use_silu &&
                      (sh->hidden_type == c.hidden_type || shared_out) && sh->gate_type == c.gate_type && sh->up_type == c.up_type &&
                      sh->down_type == c.down_type && sh->gu_soa == m->gu_soa && sh->down_layout == m->down_layout;
    if (shared_out && !fuse) { set_error("moe_forward_ep: the shared expert cannot ride in the routed launches"); return KTB200_EINVAL; }
    if (fuse) { rp.x0 = sh->gate; rp.x1 = sh->up; rp.shared_token = shared_token; }
    int rc = launch_rows<true>(fg, rp, qlen, m->device, s);
    if (rc) return rc;
    if (mid) KTB_CUDA_CHECK(cudaEventRecord(mid, s));

    ReduceParams dp{};
    dp.shared_token = -1;
    dp.w = c.down_proj; dp.type = c.down_type; dp.n_experts = c.expert_num; dp.rows = c.hidden_size;
    dp.ncols = c.intermediate_size; dp.slots = k; dp.ids = ids; dp.id_offset = c.expert_id_offset;
    dp.weights = weights; dp.a = m->inter; dp.out = output; dp.hidden_type = out_type; dp.accumulate = 0; dp.bsz = bsz;
    if (fuse) { dp.xw = sh->down; dp.shared_token = shared_token; dp.xw_out = shared_out; dp.xw_out_type = sh->hidden_type; }
    rc = launch_reduce(fd, dp, qlen, m->device, s);
    if (rc || !sh || fuse) return rc;
    return ktb200_mlp_forward(const_cast<ktb200_mlp*>(sh), qlen, input, output, 1, bsz, (void*)s);
}

int ktb200_moe_forward_shared(ktb200_moe* m, ktb200_mlp* shared, int qlen, int k, const int64_t* ids, const float* weights,
                              const void* input, void* output, const int* bsz, void* stream) {
    if (shared && !shared->loaded) { set_error("shared expert: Not Loaded"); return KTB200_ESTATE; }
    return moe_forward_impl(m, qlen, k, ids, weights, input, output, bsz, (cudaStream_t)stream, nullptr, shared);
}

int ktb200_moe_forward_ep(ktb200_moe* m, ktb200_mlp* shared, int qlen, int k, const int64_t* ids, const float* weights,
                          const void* input, void* partial_out, int own_token, void* shared_out, const int* bsz, void* stream) {
    if (!shared || !shared_out || own_token < 0 || own_token >= qlen) { set_error("moe_forward_ep: shared handle, shared_out and 0 <= own_token < qlen are required"); return KTB200_EINVAL; }
    if (!shared->loaded) { set_error("shared expert: Not Loaded"); return KTB200_ESTATE; }
    if (m && is_rawint4(m->cfg.gate_type)) { set_error("moe_forward_ep: RAWINT4_G32 experts are not supported (their kernels have no shared-expert slot)"); return KTB200_EINVAL; }
    if (m) for (int t : {m->cfg.gate_type, m->cfg.up_type, m->cfg.down_type})
        if (is_iquant(t)) { set_error("moe_forward_ep: %s experts are not supported (expert parallelism does not take the i-quants)", iquant_name(t)); return KTB200_EINVAL; }
    // shared_out rows are indexed like the tokens: point the kernels at a virtual base so that row `own_token` is shared_out
    uint8_t* base = reinterpret_cast<uint8_t*>(shared_out) - (size_t)own_token * shared->H * type_size(shared->hidden_type);
    return moe_forward_impl(m, qlen, k, ids, weights, input, partial_out, bsz, (cudaStream_t)stream, nullptr, shared, own_token, base);
}

int ktb200_moe_forward(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input,
                       void* output, const int* bsz, void* stream) {
    return moe_forward_impl(m, qlen, k, ids, weights, input, output, bsz, (cudaStream_t)stream, nullptr);
}

// the shard step of ktb200_moe_ep_forward_tokens (ep_tokens.cu): the routed sums of this handle's experts, unrounded fp32
extern "C++" {
namespace ktb {
int moe_forward_f32_out(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input, float* output,
                        cudaStream_t s) {
    return moe_forward_impl(m, qlen, k, ids, weights, input, output, nullptr, s, nullptr, nullptr, -1, nullptr, KTB200_TYPE_F32);
}
}  // namespace ktb
}

int ktb200_moe_forward_timed(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input,
                             void* output, void* stream, float* ms_gate_up, float* ms_down) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    DeviceGuard g(m->device);
    cudaStream_t s = (cudaStream_t)stream;
    cudaEvent_t e0, e1, e2;
    KTB_CUDA_CHECK(cudaEventCreate(&e0));
    KTB_CUDA_CHECK(cudaEventCreate(&e1));
    KTB_CUDA_CHECK(cudaEventCreate(&e2));
    KTB_CUDA_CHECK(cudaEventRecord(e0, s));
    int rc = moe_forward_impl(m, qlen, k, ids, weights, input, output, nullptr, s, e1);
    if (rc == KTB200_OK) {
        cudaEventRecord(e2, s);
        cudaError_t e = cudaEventSynchronize(e2);
        if (e != cudaSuccess) { set_error("timed forward: %s", cudaGetErrorString(e)); rc = KTB200_ECUDA; }
        else {
            if (ms_gate_up) cudaEventElapsedTime(ms_gate_up, e0, e1);
            if (ms_down) cudaEventElapsedTime(ms_down, e1, e2);
        }
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(e2);
    return rc;
}

int ktb200_moe_warm_up(ktb200_moe* m, void* stream) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    if (!m->loaded) { set_error("Not Loaded"); return KTB200_ESTATE; }
    DeviceGuard g(m->device);
    const ktb200_moe_config& c = m->cfg;
    cudaStream_t s = (cudaStream_t)stream;
    // zero input, weight 0, every expert once (moe.cpp:119-132)
    KTB_CUDA_CHECK(cudaMemsetAsync(m->in_d, 0, (size_t)c.hidden_size * type_size(c.hidden_type), s));
    KTB_CUDA_CHECK(cudaMemsetAsync(m->w_d, 0, sizeof(float), s));
    for (int e = 0; e < c.expert_num; e++) {
        const int64_t id = e + c.expert_id_offset;
        KTB_CUDA_CHECK(cudaMemcpyAsync(m->ids_d, &id, sizeof(id), cudaMemcpyHostToDevice, s));
        KTB_CUDA_CHECK(cudaStreamSynchronize(s));
        int rc = ktb200_moe_forward(m, 1, 1, m->ids_d, m->w_d, m->in_d, m->out_d, nullptr, stream);
        if (rc) return rc;
    }
    KTB_CUDA_CHECK(cudaStreamSynchronize(s));
    return KTB200_OK;
}

int ktb200_moe_forward_host(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input,
                            void* output, void* stream) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    if (qlen <= 0) return KTB200_OK;
    const ktb200_moe_config& c = m->cfg;
    if (qlen > c.group_max_len || k <= 0 || k > c.routed_expert_num) { set_error("forward_host: qlen/k out of range"); return KTB200_EINVAL; }
    DeviceGuard g(m->device);
    cudaStream_t s = (cudaStream_t)stream;
    const size_t hid = (size_t)qlen * c.hidden_size * type_size(c.hidden_type);
    KTB_CUDA_CHECK(cudaMemcpyAsync(m->ids_d, ids, (size_t)qlen * k * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    KTB_CUDA_CHECK(cudaMemcpyAsync(m->w_d, weights, (size_t)qlen * k * sizeof(float), cudaMemcpyHostToDevice, s));
    KTB_CUDA_CHECK(cudaMemcpyAsync(m->in_d, input, hid, cudaMemcpyHostToDevice, s));
    int rc = ktb200_moe_forward(m, qlen, k, m->ids_d, m->w_d, m->in_d, m->out_d, nullptr, stream);
    if (rc) return rc;
    KTB_CUDA_CHECK(cudaMemcpyAsync(output, m->out_d, hid, cudaMemcpyDeviceToHost, s));
    KTB_CUDA_CHECK(cudaStreamSynchronize(s));
    return KTB200_OK;
}

// ------------------------------------------------------------------------------------------ linear
struct ktb200_linear {
    int in_size, out_size, proj_type, hidden_type, group_max_len, device;
    const void* proj;
    bool loaded, soa;
};

int ktb200_linear_create(int in_size, int out_size, const void* proj, int proj_type, int hidden_type, int group_max_len,
                         int device, ktb200_linear** out) {
    if (!out || !proj) { set_error("null argument"); return KTB200_EINVAL; }
    if (is_iquant(proj_type)) { set_error("LinearConfig: %s is a routed-expert type; linears take Q2_K..Q6_K and IQ4_XS", iquant_name(proj_type)); return KTB200_EINVAL; }
    if (!weight_type_ok(proj_type)) { set_error("LinearConfig: unsupported ggml type %d", proj_type); return KTB200_EINVAL; }
    if (!is_hidden_type(hidden_type)) { set_error("LinearConfig: bad hidden_type %d", hidden_type); return KTB200_EINVAL; }
    if (in_size <= 0 || out_size <= 0 || in_size % QK_K) { set_error("LinearConfig: input_size %d must be a positive multiple of 256", in_size); return KTB200_EINVAL; }
    ktb200_linear* l = new (std::nothrow) ktb200_linear();
    if (!l) return KTB200_ENOMEM;
    l->in_size = in_size; l->out_size = out_size; l->proj = proj; l->proj_type = proj_type; l->hidden_type = hidden_type;
    l->group_max_len = group_max_len; l->device = device; l->loaded = false; l->soa = false;
    *out = l;
    return KTB200_OK;
}
void ktb200_linear_destroy(ktb200_linear* l) { delete l; }

int ktb200_linear_load_weights(ktb200_linear* l, void* stream) {
    if (!l) { set_error("null handle"); return KTB200_EINVAL; }
    if (l->loaded) return KTB200_OK;
    DeviceGuard g(l->device);
    if (l->proj_type == KTB200_TYPE_Q6_K && l->out_size % 8 == 0 && (size_t)8 * SZ_Q6_K * (l->in_size / QK_K) <= 200 * 1024) {
        int rc = repack_q6k(const_cast<void*>(l->proj), l->out_size, l->in_size, l->device, (cudaStream_t)stream);
        if (rc) return rc;
        l->soa = true;
    }
    l->loaded = true;
    return KTB200_OK;
}

int ktb200_linear_forward(ktb200_linear* l, int qlen, const void* input, void* output, const float* bias, const int* bsz,
                          void* stream) {
    if (!l) { set_error("null handle"); return KTB200_EINVAL; }
    if (!l->loaded) { set_error("Not Loaded"); return KTB200_ESTATE; }
    if (qlen <= 0) return KTB200_OK;
    if (!input || !output) { set_error("forward: null pointer"); return KTB200_EINVAL; }
    DeviceGuard g(l->device);
    RowsParams rp{};
    rp.shared_token = -1;
    rp.w0 = l->proj; rp.w1 = nullptr; rp.type0 = rp.type1 = l->proj_type; rp.n_experts = 1; rp.rows = l->out_size;
    rp.ncols = l->in_size; rp.slots = 1; rp.ids = nullptr; rp.id_offset = 0; rp.x = input; rp.hidden_type = l->hidden_type;
    rp.use_silu = 0; rp.out_f32 = nullptr; rp.out_hidden = output; rp.bias = bias; rp.bsz = bsz;
    return launch_rows<false>(pick_fmt(l->proj_type, l->soa), rp, qlen, l->device, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------ mlp

int ktb200_mlp_create(int H, int I, const void* gate, const void* up, const void* down, int gate_type, int up_type,
                      int down_type, int hidden_type, int group_max_len, int device, ktb200_mlp** out) {
    if (!out || !gate || !up || !down) { set_error("null argument"); return KTB200_EINVAL; }
    for (int t : {gate_type, up_type, down_type})
        if (is_iquant(t)) { set_error("MLPConfig: %s is a routed-expert type; MLPs take Q2_K..Q6_K and IQ4_XS", iquant_name(t)); return KTB200_EINVAL; }
    if (!weight_type_ok(gate_type) || !weight_type_ok(up_type) || !weight_type_ok(down_type)) { set_error("MLPConfig: unsupported ggml type"); return KTB200_EINVAL; }
    if (!is_hidden_type(hidden_type)) { set_error("MLPConfig: bad hidden_type"); return KTB200_EINVAL; }
    if (H <= 0 || I <= 0 || H % QK_K || I % QK_K || group_max_len <= 0) { set_error("MLPConfig: sizes must be positive multiples of 256"); return KTB200_EINVAL; }
    DeviceGuard g(device);
    ktb200_mlp* m = new (std::nothrow) ktb200_mlp();
    if (!m) return KTB200_ENOMEM;
    m->H = H; m->I = I; m->gate = gate; m->up = up; m->down = down; m->gate_type = gate_type; m->up_type = up_type;
    m->down_type = down_type; m->hidden_type = hidden_type; m->group_max_len = group_max_len; m->device = device;
    m->loaded = m->gu_soa = false; m->down_layout = LAYOUT_RAW; m->inter = nullptr;
    if (cudaMalloc(&m->inter, (size_t)group_max_len * I * sizeof(float)) != cudaSuccess) {
        set_error("cudaMalloc failed");
        delete m;
        return KTB200_ENOMEM;
    }
    *out = m;
    return KTB200_OK;
}
void ktb200_mlp_destroy(ktb200_mlp* m) {
    if (!m) return;
    DeviceGuard g(m->device);
    cudaFree(m->inter);
    delete m;
}
int ktb200_mlp_load_weights(ktb200_mlp* m, void* stream) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    if (m->loaded) return KTB200_OK;
    DeviceGuard g(m->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (m->gate_type == KTB200_TYPE_Q6_K && m->up_type == KTB200_TYPE_Q6_K && m->I % 8 == 0) {
        int rc = repack_q6k(const_cast<void*>(m->gate), m->I, m->H, m->device, s);
        if (rc) return rc;
        rc = repack_q6k(const_cast<void*>(m->up), m->I, m->H, m->device, s);
        if (rc) return rc;
        m->gu_soa = true;
    }
    // 17 slots: a shared expert stays fusable with up to 16 routed experts per token (ktb200_moe_forward_shared)
    if (m->down_type == KTB200_TYPE_Q6_K && q6k4t_eligible(m->H, m->I, 17, m->device)) {
        int rc = repack_q6k4t(const_cast<void*>(m->down), m->H, m->I, m->device, s);
        if (rc) return rc;
        m->down_layout = LAYOUT_T4;
    } else if (m->down_type == KTB200_TYPE_Q6_K && m->H % 8 == 0 && (size_t)8 * SZ_Q6_K * (m->I / QK_K) <= 200 * 1024) {
        int rc = repack_q6k(const_cast<void*>(m->down), m->H, m->I, m->device, s);
        if (rc) return rc;
        m->down_layout = LAYOUT_SOA8;
    }
    m->loaded = true;
    return KTB200_OK;
}
int ktb200_mlp_forward(ktb200_mlp* m, int qlen, const void* input, void* output, int accumulate, const int* bsz, void* stream) {
    if (!m) { set_error("null handle"); return KTB200_EINVAL; }
    if (!m->loaded) { set_error("Not Loaded"); return KTB200_ESTATE; }
    if (qlen <= 0) return KTB200_OK;
    if (qlen > m->group_max_len) { set_error("forward: qlen=%d exceeds group_max_len=%d", qlen, m->group_max_len); return KTB200_EINVAL; }
    DeviceGuard g(m->device);
    cudaStream_t s = (cudaStream_t)stream;
    FmtId fg = pick_fmt(m->gate_type, m->gu_soa), fu = pick_fmt(m->up_type, m->gu_soa);
    if (fg != fu) fg = fu = FMT_GENK;
    RowsParams rp{};
    rp.shared_token = -1;
    rp.w0 = m->gate; rp.w1 = m->up; rp.type0 = m->gate_type; rp.type1 = m->up_type; rp.n_experts = 1; rp.rows = m->I;
    rp.ncols = m->H; rp.slots = 1; rp.ids = nullptr; rp.x = input; rp.hidden_type = m->hidden_type; rp.use_silu = 1;
    rp.out_f32 = m->inter; rp.bsz = bsz;
    int rc = launch_rows<true>(fg, rp, qlen, m->device, s);
    if (rc) return rc;
    ReduceParams dp{};
    dp.shared_token = -1;
    dp.w = m->down; dp.type = m->down_type; dp.n_experts = 1; dp.rows = m->H; dp.ncols = m->I; dp.slots = 1; dp.ids = nullptr;
    dp.weights = nullptr; dp.a = m->inter; dp.out = output; dp.hidden_type = m->hidden_type; dp.accumulate = accumulate; dp.bsz = bsz;
    return launch_reduce(pick_fmt(m->down_type, m->down_layout), dp, qlen, m->device, s);
}

// ------------------------------------------------------------------------------------------ RAWINT4 pack
int ktb200_rawint4_pack(const int32_t* packed, const uint16_t* scale, long n_rows, long n_cols, void* out, void* stream) {
    if (!packed || !scale || !out) { set_error("rawint4_pack: null pointer"); return KTB200_EINVAL; }
    if (n_rows < 0 || n_cols <= 0 || n_cols % QK_K) { set_error("rawint4_pack: n_cols=%ld must be a positive multiple of 256", n_cols); return KTB200_EINVAL; }
    if ((uintptr_t)out & 15) { set_error("rawint4_pack: out must be 16-byte aligned"); return KTB200_EINVAL; }
    const long n_sb = n_rows * (n_cols / QK_K);
    if (n_sb == 0) return KTB200_OK;
    int dev = 0;
    KTB_CUDA_CHECK(cudaGetDevice(&dev));
    long blocks = (n_sb * 9 + 255) / 256;
    if (blocks > (long)num_sms(dev) * 16) blocks = (long)num_sms(dev) * 16;
    rawint4_pack_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint32_t*>(packed), scale, n_sb,
                                                                             (int)(n_cols / QK_K), reinterpret_cast<uint4*>(out));
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

// ------------------------------------------------------------------------------------------ quantize API
int ktb200_quantize_activations(const void* x, int hidden_type, long n_rows, long n_cols, int act_type, void* out, void* stream) {
    if (!x || !out) { set_error("null pointer"); return KTB200_EINVAL; }
    if (!is_hidden_type(hidden_type)) { set_error("bad hidden_type %d", hidden_type); return KTB200_EINVAL; }
    const long n = n_rows * n_cols;
    cudaStream_t s = (cudaStream_t)stream;
    if (act_type == KTB200_TYPE_Q8_K) {
        if (n_cols % QK_K) { set_error("Q8_K needs n_cols %% 256 == 0"); return KTB200_EINVAL; }
        const long nb = n / QK_K;
        if (nb == 0) return KTB200_OK;
        quantize_q8k_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, s>>>(x, hidden_type, nb, reinterpret_cast<uint8_t*>(out));
    } else if (act_type == KTB200_TYPE_Q8_0) {
        if (n_cols % 32) { set_error("Q8_0 needs n_cols %% 32 == 0"); return KTB200_EINVAL; }
        const long nb = n / 32;
        if (nb == 0) return KTB200_OK;
        quantize_q8_0_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, s>>>(x, hidden_type, nb, reinterpret_cast<uint8_t*>(out));
    } else {
        set_error("activation type %d is not a vec_dot type", act_type);
        return KTB200_EINVAL;
    }
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

}  // extern "C"
