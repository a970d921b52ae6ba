/*
 *  exact_wgmma.cu — brute-force search over i8 vectors on Hopper's warpgroup tensor cores.
 *
 *  Same contract and the same bits as exact_imma.cu (integer sums are exact in any order: the three i8 metrics are functions
 *  of the integer triple (ab, a2, b2), index_plugins.hpp:1914-1916 / simsimd spatial.h:1880-1972 / dot.h:1749-1775), but the
 *  contraction runs as asynchronous `wgmma.mma_async ... s32.s8.s8` with both operands read from shared memory written by
 *  TMA tensor copies (SASS: HGMMA.IMMA / UTMALDG), instead of warp-level `mma.sync`.
 *
 *  One CTA = one tile of 128 queries against one segment of the stored vectors, walked in tiles of 256 vectors:
 *      warp 8        TMA producer (its warpgroup gives most of its registers to the consumers, setmaxnreg): per k-block of 128 bytes one box of the query tile (128 rows) and one of the vector tile
 *                    (256 rows) into a 4-stage ring of 128B-swizzled shared memory, `full` / `empty` mbarriers
 *      warps 0..7    two consumer warpgroups, one per half of the query tile. Each issues four M64 x N256 x K32 wgmma per
 *                    k-block into 128 s32 accumulators per thread and frees the stage once the group has completed. After
 *                    the last k-block every thread holds two rows x 64 columns of the tile: it turns each integer dot
 *                    product into the metric's float (i8_distance, shared with the IMMA kernel) only for columns that pass a
 *                    conservative integer filter against the row's current worst, and — rarely — inserts into that row's
 *                    k-best list under (distance ascending, slot descending). The four threads that share a row take turns,
 *                    so a list has one writer at a time. The lists live in SHARED memory (count <= 24; larger counts take the
 *                    mma.sync kernel). While one warpgroup filters, the other's MMAs keep the tensor cores busy.
 *  The per-(query, segment) lists are merged by exact_merge_kernel exactly as for the other scan kernels.
 */
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "device_index.h"
#include "exact_args.h"
#include "exact_i8.h"
#include "warp_primitives.cuh"

namespace usearch_b200 {

namespace {

constexpr int WG_BM = 128;      /* queries per CTA: two warpgroups of 64 rows (the M of the instruction) */
constexpr int WG_BN = 256;      /* stored vectors per tile: the N of the instruction */
constexpr int WG_BK = 128;      /* bytes of K per stage: one 128-byte swizzle row */
constexpr int WG_K = 32;        /* K of one s8 instruction */
constexpr int WG_STAGES = 4;
constexpr int WG_A_BYTES = WG_BM * WG_BK, WG_B_BYTES = WG_BN * WG_BK, WG_STAGE_BYTES = WG_A_BYTES + WG_B_BYTES; /* 48 KB */
constexpr int WG_CONSUMERS = 256;                 /* warps 0..7: two warpgroups */
constexpr int WG_THREADS = WG_CONSUMERS + 128;    /* + warpgroup 2, whose first lane issues the TMA copies */
constexpr int WG_PRODUCER_REGS = 40, WG_CONSUMER_REGS = 232; /* setmaxnreg: 128 x 40 + 256 x 232 <= 64 K registers */
constexpr int WG_KMAX = 24;        /* k-best lists of up to this many entries live in shared memory (row stride 25 words) */
constexpr int WG_LIST_STRIDE = WG_KMAX + 1;
constexpr int WG_LIST_BYTES = WG_BM * WG_LIST_STRIDE * 8;

__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }

/* shared-memory matrix descriptor of a K-major operand tile written by TMA with the 128-byte swizzle (PTX ISA, "Matrix
 * Descriptor Format" of wgmma): start address >> 4 in [0,14), leading-dimension offset (unused by this layout, 1) in
 * [16,30), stride between groups of 8 rows = 1024 B >> 4 in [32,46), layout SWIZZLE_128B = 1 in [62,64) */
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
    uint64_t desc = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    desc |= (uint64_t)1 << 16;
    desc |= (uint64_t)(1024u >> 4) << 32;
    desc |= (uint64_t)1 << 62;
    return desc;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

/* D[64 x 256] += A[64 x 32] * B[256 x 32]^T, s8 x s8 -> s32, both operands K-major in shared memory */
__device__ __forceinline__ void wgmma_i8(int (&d)[128], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
        "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, "
        "%74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, "
        "%98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, "
        "%118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, 1;"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]),
          "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]),
          "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]),
          "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]),
          "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]),
          "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]),
          "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
          "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]),
          "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]),
          "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]),
          "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]),
          "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]),
          "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]),
          "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]),
          "+r"(d[127])
        : "l"(a_desc), "l"(b_desc)
        : "memory");
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, CUtensorMap const* map, uint32_t x, uint32_t y, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(map), "r"(x), "r"(y), "r"(bar)
                 : "memory");
}

/* one thread, one list: sorted insert under (distance ascending, slot descending), the order a sequence of
 * sorted_buffer_gt::insert calls in slot order converges to (search_exact_, index.hpp:4251-4268) */
__device__ __noinline__ void list_insert(float* ld, uint32_t* ls, uint32_t& size, uint32_t k, float cd, uint32_t cs) {
    uint32_t pos = size;
    while (pos > 0) { /* entries that sort after the candidate move one place to the right */
        float const d = ld[pos - 1];
        if (d < cd || (d == cd && ls[pos - 1] > cs)) break;
        --pos;
    }
    if (pos >= k) return;
    uint32_t const new_size = size < k ? size + 1 : k;
    for (uint32_t i = new_size - 1; i > pos; --i) { ld[i] = ld[i - 1]; ls[i] = ls[i - 1]; }
    ld[pos] = cd;
    ls[pos] = cs;
    size = new_size;
}

/* what one query row needs to filter and insert: its norm terms and the filter's thresholds (exact_i8.h, where their
 * soundness is derived) from the list's worst */
template <uint32_t METRIC> struct row_t {
    uint32_t row;  /* 0..127 in the tile */
    bool live;
    int qa2;
    float qr;
    i8_filter_t<METRIC> filter;

    __device__ __forceinline__ void thresholds(uint32_t size, uint32_t k, float worst) { filter.set_thresholds(size, k, worst, qa2, qr); }
};

/* accumulator layout of m64nNk32 (PTX ISA, wgmma "Matrix fragments for D"): warp w of the warpgroup, lane l holds, for column
 * block j = 0..31, d[4j + e] at (row 16w + l/4, column 8j + 2(l%4) + e) and d[4j + 2 + e] at row + 8, e = 0, 1.
 * H selects the row: bit 2j + e of the returned mask flags column 8j + 2(l%4) + e. */
template <uint32_t METRIC, int H>
__device__ __forceinline__ uint64_t filter_row(int const (&d)[128], row_t<METRIC> const& r, int const* b2, float const* rn,
                                               uint32_t const* mask, uint32_t col0) {
    uint64_t pm = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            uint32_t const col = 8u * j + col0 + e;
            int const v = d[4 * j + 2 * H + e];
            bool maybe = r.filter.maybe(v, METRIC == METRIC_L2SQ ? b2[col] : 0, METRIC == METRIC_COS ? rn[col] : 0.f);
            maybe = maybe && ((mask[j >> 2] >> (col & 31u)) & 1u);
            pm |= maybe ? (1ull << (2 * j + e)) : 0ull;
        }
    }
    return r.live ? pm : 0ull;
}

/* the exact metric and the sorted insert for the flagged columns of one row; the caller is the row's only writer */
template <uint32_t METRIC, bool SWAP, int H>
__device__ __forceinline__ void insert_row(int const (&d)[128], row_t<METRIC> const& r, uint64_t pm, int const* b2, float const* rn,
                                           uint32_t col0, uint32_t tile_base, uint32_t k, float* ld, uint32_t* ls, uint32_t* row_size) {
    uint32_t size = row_size[r.row];
    float worst = size == k ? ld[k - 1] : 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            if (!((pm >> (2 * j + e)) & 1ull)) continue;
            uint32_t const col = 8u * j + col0 + e;
            float const dist = i8_distance<METRIC, SWAP>(d[4 * j + 2 * H + e], r.qa2, b2[col], r.qr, rn[col]);
            if (size < k || !(dist > worst)) {
                list_insert(ld, ls, size, k, dist, tile_base + col);
                if (size == k) worst = ld[k - 1];
            }
        }
    }
    row_size[r.row] = size;
}

template <uint32_t METRIC, bool SWAP>
__global__ void __launch_bounds__(WG_THREADS, 1) exact_wgmma_kernel(__grid_constant__ device_index_t const ix,
                                                                    __grid_constant__ exact_args_t const a,
                                                                    __grid_constant__ CUtensorMap const map_queries,
                                                                    __grid_constant__ CUtensorMap const map_vectors) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bars[2 * WG_STAGES];
    __shared__ int col_b2[2][WG_BN];             /* per warpgroup: sum of squares of the tile's vectors */
    __shared__ float col_rn[2][WG_BN];           /* cos: their reciprocal norms */
    __shared__ uint32_t col_mask[2][WG_BN / 32]; /* usable columns: inside the segment and not removed */
    __shared__ uint32_t row_size[WG_BM];         /* entries in each row's list */

    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t const stages = (smem_u32(smem_raw) + 1023u) & ~1023u; /* the swizzle atom is 1024 bytes */
    uint32_t const full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[WG_STAGES]);
    uint32_t const vs = (uint32_t)ix.vec_stride, nkb = (vs + WG_BK - 1) / WG_BK;
    uint32_t const q0 = blockIdx.x * WG_BM;
    uint32_t const seg_lo = blockIdx.y * a.segment_len, seg_hi = min(ix.n, seg_lo + a.segment_len);
    uint32_t const ntiles = seg_hi > seg_lo ? (seg_hi - seg_lo + WG_BN - 1) / WG_BN : 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < WG_STAGES; ++s) { mbar_init(full0 + 8u * s, 1); mbar_init(empty0 + 8u * s, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (threadIdx.x < WG_BM) row_size[threadIdx.x] = 0;
    __syncthreads();

    if (threadIdx.x >= WG_CONSUMERS) {
        /* ===== TMA producer ===== */
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WG_PRODUCER_REGS));
        if (threadIdx.x == WG_CONSUMERS) {
            uint32_t stage = 0, phase = 0;
            for (uint32_t t = 0; t < ntiles; ++t) {
                uint32_t const tile_base = seg_lo + t * WG_BN;
                for (uint32_t kb = 0; kb < nkb; ++kb) {
                    mbar_wait(empty0 + 8u * stage, phase ^ 1u);
                    uint32_t const sa = stages + stage * WG_STAGE_BYTES, sb = sa + WG_A_BYTES;
                    mbar_expect_tx(full0 + 8u * stage, WG_STAGE_BYTES);
                    tma_load_2d(sa, &map_queries, kb * WG_BK, q0, full0 + 8u * stage);
                    tma_load_2d(sb, &map_vectors, kb * WG_BK, tile_base, full0 + 8u * stage);
                    if (++stage == WG_STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
        return;
    }

    /* ===== consumers: warpgroup g owns query rows 64g .. 64g+63 of the tile ===== */
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WG_CONSUMER_REGS));
    uint32_t const g = threadIdx.x >> 7, wt = threadIdx.x & 127u;
    uint32_t const col0 = 2u * ((uint32_t)lane & 3u), quad = (uint32_t)lane & 3u;
    row_t<METRIC> rows[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        rows[h].row = g * 64u + (uint32_t)(warp & 3) * 16u + ((uint32_t)lane >> 2) + 8u * h;
        uint32_t const qi = q0 + rows[h].row;
        rows[h].live = qi < a.nq;
        rows[h].qa2 = (METRIC != METRIC_IP && rows[h].live) ? a.query_norms[qi] : 0;
        rows[h].qr = METRIC == METRIC_COS ? i8_rnorm(rows[h].qa2) : 0.f;
        rows[h].thresholds(0, a.k, 0.f);
    }
    float* const ld_base = reinterpret_cast<float*>(smem_raw + (stages - smem_u32(smem_raw)) + WG_STAGES * WG_STAGE_BYTES);
    uint32_t* const ls_base = reinterpret_cast<uint32_t*>(ld_base + WG_BM * WG_LIST_STRIDE);
    int* const b2 = col_b2[g];
    float* const rn = col_rn[g];
    uint32_t* const mask = col_mask[g];

    uint32_t stage = 0, phase = 0;
    for (uint32_t t = 0; t < ntiles; ++t) {
        uint32_t const tile_base = seg_lo + t * WG_BN;
        /* per-column facts of this tile (two columns per thread), while the first operands arrive */
        for (uint32_t c = wt; c < (uint32_t)WG_BN; c += 128) {
            uint32_t const slot = tile_base + c;
            bool usable = slot < seg_hi;
            if (usable && ix.deleted_bits) usable = !((ix.deleted_bits[slot >> 5] >> (slot & 31)) & 1u);
            int const vb2 = (METRIC != METRIC_IP && slot < seg_hi) ? a.vector_norms[slot] : 0;
            b2[c] = vb2;
            rn[c] = METRIC == METRIC_COS ? i8_rnorm(vb2) : 0.f;
            uint32_t const m = __ballot_sync(0xffffffffu, usable);
            if (lane == 0) mask[c >> 5] = m;
        }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); /* this warpgroup only */

        int d[128];
#pragma unroll
        for (int i = 0; i < 128; ++i) d[i] = 0;
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < nkb; ++kb) {
            mbar_wait(full0 + 8u * stage, phase);
            uint32_t const sa = stages + stage * WG_STAGE_BYTES + g * (WG_A_BYTES / 2), sb = stages + stage * WG_STAGE_BYTES + WG_A_BYTES;
            uint64_t const da = wgmma_desc(sa), db = wgmma_desc(sb);
            wgmma_fence();
#pragma unroll
            for (uint32_t k = 0; k < WG_BK / WG_K; ++k) /* 32 bytes further along the swizzled row: +2 in the address field */
                wgmma_i8(d, da + (uint64_t)(k * WG_K >> 4), db + (uint64_t)(k * WG_K >> 4));
            wgmma_commit();
            wgmma_wait<1>(); /* the previous k-block's group has read its stage */
            if (kb > 0 && wt == 0) mbar_arrive(empty0 + 8u * prev);
            prev = stage;
            if (++stage == WG_STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        if (nkb > 0 && wt == 0) mbar_arrive(empty0 + 8u * prev);

        /* FILTER, branch-free: which columns could still enter the row's list? A conservative test on the integer dot
         * product (never misses a candidate, may flag a few too many) */
        uint64_t const pm0 = filter_row<METRIC, 0>(d, rows[0], b2, rn, mask, col0);
        uint64_t const pm1 = filter_row<METRIC, 1>(d, rows[1], b2, rn, mask, col0);
        if (__any_sync(0xffffffffu, (pm0 | pm1) != 0ull)) { /* rare once the lists are full */
            for (uint32_t turn = 0; turn < 4; ++turn) { /* the four threads of a row, one after the other */
                if (quad == turn) {
                    if (pm0) insert_row<METRIC, SWAP, 0>(d, rows[0], pm0, b2, rn, col0, tile_base, a.k, ld_base + rows[0].row * WG_LIST_STRIDE,
                                                         ls_base + rows[0].row * WG_LIST_STRIDE, row_size);
                    if (pm1) insert_row<METRIC, SWAP, 1>(d, rows[1], pm1, b2, rn, col0, tile_base, a.k, ld_base + rows[1].row * WG_LIST_STRIDE,
                                                         ls_base + rows[1].row * WG_LIST_STRIDE, row_size);
                }
                __syncwarp();
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint32_t const size = row_size[rows[h].row];
                rows[h].thresholds(size, a.k, size == a.k ? ld_base[rows[h].row * WG_LIST_STRIDE + a.k - 1] : 0.f);
            }
        }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); /* nobody overwrites col_* before all have read them */
    }
    __syncwarp();
    if (quad < 2 && rows[quad].live) { /* the row's list -> the per-(query, segment) partial result */
        row_t<METRIC> const& r = rows[quad];
        uint32_t const qi = q0 + r.row, size = row_size[r.row];
        size_t const list = ((size_t)qi * a.segments + blockIdx.y) * a.k;
        for (uint32_t i = 0; i < size; ++i) {
            a.part_d[list + i] = ld_base[r.row * WG_LIST_STRIDE + i];
            a.part_s[list + i] = ls_base[r.row * WG_LIST_STRIDE + i];
        }
        a.part_n[(size_t)qi * a.segments + blockIdx.y] = size;
    }
}

/* cuTensorMapEncodeTiled through the runtime's driver entry point: the library links no libcuda */
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, cuuint64_t const*, cuuint64_t const*,
                                    cuuint32_t const*, cuuint32_t const*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

encode_tiled_fn encode_tiled() {
    static encode_tiled_fn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return reinterpret_cast<encode_tiled_fn>(p);
    }();
    return fn;
}

/* a row-major byte matrix [rows x row_bytes], rows `pitch` bytes apart, read in boxes of 128 bytes x box_rows with the 128-byte
 * swizzle; bytes and rows outside the matrix arrive as zeros (which add nothing to a dot product) */
bool make_map(CUtensorMap* map, void const* base, uint64_t rows, uint64_t row_bytes, uint64_t pitch, uint32_t box_rows) {
    encode_tiled_fn fn = encode_tiled();
    if (!fn) return false;
    cuuint64_t dims[2] = {row_bytes, rows};
    cuuint64_t strides[1] = {pitch};
    cuuint32_t box[2] = {(cuuint32_t)WG_BK, box_rows};
    cuuint32_t elem[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, elem, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <uint32_t METRIC, bool SWAP>
cudaError_t wgmma_launch_t(exact_args_t const& a, device_index_t const& ix, dim3 grid, CUtensorMap const& mq, CUtensorMap const& mv,
                           cudaStream_t stream) {
    size_t const smem = exact_wgmma_smem_bytes();
    cudaError_t e = cudaFuncSetAttribute(exact_wgmma_kernel<METRIC, SWAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    exact_wgmma_kernel<METRIC, SWAP><<<grid, WG_THREADS, smem, stream>>>(ix, a, mq, mv);
    return cudaGetLastError();
}

template <uint32_t METRIC>
cudaError_t wgmma_launch_t(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, CUtensorMap const& mq, CUtensorMap const& mv,
                           cudaStream_t stream) {
    return swap ? wgmma_launch_t<METRIC, true>(a, ix, grid, mq, mv, stream) : wgmma_launch_t<METRIC, false>(a, ix, grid, mq, mv, stream);
}

} // namespace

size_t exact_wgmma_smem_bytes() { return (size_t)WG_STAGES * WG_STAGE_BYTES + 1024 + WG_LIST_BYTES; }
int exact_wgmma_tile_queries() { return WG_BM; }
int exact_wgmma_tile_vectors() { return WG_BN; }

/* false when the driver cannot encode tensor maps or the operands are not laid out for them: the caller takes the IMMA kernel */
bool exact_wgmma_usable(device_index_t const& ix, exact_args_t const& a) {
    return a.k <= (uint32_t)WG_KMAX && encode_tiled() != nullptr && (reinterpret_cast<uintptr_t>(ix.vectors) & 15) == 0 &&
           (reinterpret_cast<uintptr_t>(a.queries) & 15) == 0 && (a.query_stride & 15) == 0 && (ix.vec_stride & 15) == 0;
}

cudaError_t exact_wgmma_launch(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream) {
    CUtensorMap mq, mv;
    if (!make_map(&mq, a.queries, a.nq, ix.vec_stride, a.query_stride, WG_BM) || !make_map(&mv, ix.vectors, ix.n, ix.vec_stride, ix.vec_stride, WG_BN))
        return cudaErrorInvalidValue;
    switch (ix.metric) {
    case METRIC_IP: return wgmma_launch_t<METRIC_IP>(ix, a, swap, grid, mq, mv, stream);
    case METRIC_L2SQ: return wgmma_launch_t<METRIC_L2SQ>(ix, a, swap, grid, mq, mv, stream);
    case METRIC_COS: return wgmma_launch_t<METRIC_COS>(ix, a, swap, grid, mq, mv, stream);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace usearch_b200
