/*
 *  exact_imma.cu — brute-force search over i8 vectors on the tensor cores.
 *
 *  Integer sums are exact in any order, so this is the one scalar kind where a GEMM reproduces the reference
 *  bit for bit (SURVEY.md §8 N1): the three i8 metrics are functions of the integer triple
 *  (ab, a2, b2) = (sum a*b, sum a*a, sum b*b)
 *      ip    1 - float(ab)                               index_plugins.hpp:1914-1916 over simsimd_dot_i8
 *      l2sq  float(a2 + b2 - 2 ab)  == sum (a-b)^2       spatial.h l2sq_i8 (i32 accumulation)
 *      cos   normalise(float(ab), float(a2), float(b2))  spatial.h:1904-1972 -> the f32 normaliser
 *  ab comes from `mma.sync.m16n8k32.s8` (SASS IMMA.16832), a2 / b2 from one dp4a pass per operand.
 *
 *  CTA = 8 warps, tile = 128 queries x 128 stored vectors, K walked in 64-byte slices through a 5-stage cp.async
 *  pipeline (both operands streamed; the query tile stays hot in L2). Shared rows are 64 bytes, unpadded: a
 *  quarter-warp reads two whole rows = 128 contiguous bytes per LDS.128, conflict-free. One LDS.128 per row and
 *  slice feeds two k-steps: the 16 bytes a thread loads at offset 16*t are used as its (a0, a2) registers of both
 *  steps — a permutation of K applied identically to both operands, which leaves every dot product unchanged.
 *  The finished 128 x 128 distances go through shared memory (aliasing the drained pipeline) so that each warp
 *  owns 16 query rows and runs the same threshold-then-rare-insert into the per-(query, segment) k-best lists as
 *  the register-tiled kernel; exact_merge_kernel finishes.
 */
#include <cuda_runtime.h>

#include <cstdint>

#include "device_index.h"
#include "exact_args.h"
#include "exact_i8.h"
#include "metrics.cuh"
#include "warp_primitives.cuh"

namespace usearch_b200 {

namespace {

constexpr int IM_BM = 128, IM_BN = 128, IM_BK = 64, IM_STAGES = 5, IM_THREADS = 256;
constexpr int IM_STAGE_BYTES = (IM_BM + IM_BN) * IM_BK;    /* 16 KB */
constexpr int IM_DIST_STRIDE = IM_BN + 4;                  /* floats per row of the distance tile */
constexpr int IM_PIPE_BYTES = IM_STAGES * IM_STAGE_BYTES;  /* 80 KB >= 128 * 132 * 4 = 67.6 KB */
static_assert(IM_PIPE_BYTES >= IM_BM * IM_DIST_STRIDE * 4, "the distance tile aliases the pipeline stages");

__device__ __forceinline__ void cp_async16(uint32_t dst, void const* src, bool valid) {
    uint32_t const n = valid ? 16u : 0u; /* src-size 0: nothing is read, the 16 bytes are zero-filled */
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void imma_16832(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

} // namespace

/* sum of squares of every row (one warp per row): the a2 / b2 of the i8 metrics */
__global__ void i8_self_dot_kernel(uint8_t const* rows, uint64_t stride, uint32_t chunks16, uint32_t count, int* out) {
    uint32_t const row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    if (row >= count) return;
    uint4 const* v4 = reinterpret_cast<uint4 const*>(rows + (size_t)row * stride);
    int s = 0;
    for (uint32_t j = lane; j < chunks16; j += 32) {
        uint4 const x = v4[j];
        s = __dp4a((int)x.x, (int)x.x, s); s = __dp4a((int)x.y, (int)x.y, s);
        s = __dp4a((int)x.z, (int)x.z, s); s = __dp4a((int)x.w, (int)x.w, s);
    }
    s = reduce_add_i32<32>(s);
    if (lane == 0) out[row] = s;
}

/* sum of squares of the listed rows: out[j] for slot rows[j] (listed scans index the stored norms by list position) */
__global__ void i8_listed_self_dot_kernel(uint8_t const* vectors, uint64_t stride, uint32_t chunks16, uint32_t const* rows, uint32_t count,
                                          int* out) {
    uint32_t const j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    if (j >= count) return;
    uint4 const* v4 = reinterpret_cast<uint4 const*>(vectors + (size_t)rows[j] * stride);
    int s = 0;
    for (uint32_t c = lane; c < chunks16; c += 32) {
        uint4 const x = v4[c];
        s = __dp4a((int)x.x, (int)x.x, s); s = __dp4a((int)x.y, (int)x.y, s);
        s = __dp4a((int)x.z, (int)x.z, s); s = __dp4a((int)x.w, (int)x.w, s);
    }
    s = reduce_add_i32<32>(s);
    if (lane == 0) out[j] = s;
}

/* LISTED: the CTA serves work item a.items[blockIdx.x]; column j of its segment is slot a.rows[list_begin + j] and its
 * b2 is a.vector_norms[list_begin + j] (exact_args.h) */
template <uint32_t METRIC, bool SWAP, bool LISTED = false>
__global__ void __launch_bounds__(IM_THREADS, 2) exact_imma_kernel(__grid_constant__ device_index_t const ix,
                                                                   __grid_constant__ exact_args_of<LISTED> const a) {
    extern __shared__ __align__(128) uint8_t smem[];
    int const tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    int const wm = warp >> 2, wn = warp & 3; /* warp tile: rows wm*64.., columns wn*32.. */
    uint32_t const vs = (uint32_t)ix.vec_stride, nks = (vs + IM_BK - 1) / IM_BK;
    uint32_t q0 = blockIdx.x * IM_BM, q_end = 0; /* LISTED: queries from q_end on are dead rows */
    uint32_t seg_lo = blockIdx.y * a.segment_len, seg_hi = min(ix.n, seg_lo + a.segment_len);
    uint32_t const* listed_slots = nullptr;
    int const* vnorms = nullptr;
    if constexpr (LISTED) {
        exact_item_t const it = a.items[blockIdx.x];
        q0 = it.first;
        q_end = it.first + it.count;
        listed_segment(it, a.segments, blockIdx.y, IM_BN, seg_lo, seg_hi);
        listed_slots = a.rows + it.list_begin;
        vnorms = a.vector_norms + it.list_begin;
    }
    uint32_t const ntiles = seg_hi > seg_lo ? (seg_hi - seg_lo + IM_BN - 1) / IM_BN : 0;

    float* const dist = reinterpret_cast<float*>(smem); /* aliases the pipeline, used between K loops only */
    int* const qa2 = reinterpret_cast<int*>(smem + IM_PIPE_BYTES);
    int* const vb2 = qa2 + IM_BM;
    uint32_t* const rsize = reinterpret_cast<uint32_t*>(vb2 + IM_BN);
    float* const rworst = reinterpret_cast<float*>(rsize + IM_BM);
    float* const qrn = rworst + IM_BM; /* cos: reciprocal norms of the rows / columns */
    float* const vrn = qrn + IM_BM;
    uint32_t* const vmask = reinterpret_cast<uint32_t*>(vrn + IM_BN); /* 4 words: usable columns of the tile */
    uint32_t const pipe = smem_u32(smem);

    if (tid < IM_BM) {
        qa2[tid] = (METRIC != METRIC_IP && q0 + tid < (LISTED ? q_end : a.nq)) ? a.query_norms[q0 + tid] : 0;
        qrn[tid] = METRIC == METRIC_COS ? i8_rnorm(qa2[tid]) : 0.f;
        rsize[tid] = 0;
        rworst[tid] = 0.f;
    }

    auto load_slice = [&](uint32_t tile_base, uint32_t ks, uint32_t stage) {
        uint32_t const kbyte = ks * IM_BK, sbase = pipe + stage * IM_STAGE_BYTES;
#pragma unroll
        for (int i = 0; i < 2; ++i) { /* 512 chunks of the query part */
            uint32_t const c = (uint32_t)tid + (uint32_t)i * IM_THREADS, row = c >> 2, off = (c & 3u) * 16u;
            bool const ok = q0 + row < (LISTED ? q_end : a.nq) && kbyte + off < vs;
            void const* src = ok ? a.queries + (size_t)(q0 + row) * a.query_stride + kbyte + off : a.queries;
            cp_async16(sbase + row * IM_BK + off, src, ok);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) { /* 512 chunks of the stored part */
            uint32_t const c = (uint32_t)tid + (uint32_t)i * IM_THREADS, row = c >> 2, off = (c & 3u) * 16u;
            bool const ok = tile_base + row < seg_hi && kbyte + off < vs;
            void const* src = ok ? ix.vectors + (size_t)(LISTED ? listed_slots[tile_base + row] : tile_base + row) * ix.vec_stride + kbyte + off
                                 : ix.vectors;
            cp_async16(sbase + IM_BM * IM_BK + row * IM_BK + off, src, ok);
        }
    };

    for (uint32_t tile = 0; tile < ntiles; ++tile) {
        uint32_t const tile_base = seg_lo + tile * IM_BN;
        /* pipeline prologue (the previous tile's epilogue ended with a barrier) */
#pragma unroll
        for (int s = 0; s < IM_STAGES - 1; ++s) {
            if ((uint32_t)s < nks) load_slice(tile_base, (uint32_t)s, (uint32_t)s);
            cp_async_commit();
        }
        if (tid < IM_BN) { /* per-column facts of this tile */
            uint32_t const pos = tile_base + (uint32_t)tid;
            uint32_t const slot = LISTED ? (pos < seg_hi ? listed_slots[pos] : 0u) : pos;
            bool usable = pos < seg_hi;
            if (usable && ix.deleted_bits) usable = !((ix.deleted_bits[slot >> 5] >> (slot & 31)) & 1u);
            vb2[tid] = (METRIC != METRIC_IP && pos < seg_hi) ? (LISTED ? vnorms : a.vector_norms)[pos] : 0;
            vrn[tid] = METRIC == METRIC_COS ? i8_rnorm(vb2[tid]) : 0.f;
            uint32_t const m = __ballot_sync(0xffffffffu, usable);
            if (lane == 0) vmask[warp] = m;
        }

        int acc[4][4][4];
#pragma unroll
        for (int mi = 0; mi < 4; ++mi)
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[mi][ni][r] = 0;

        for (uint32_t ks = 0; ks < nks; ++ks) {
            cp_async_wait<IM_STAGES - 2>();
            __syncthreads(); /* slice ks has landed for everyone; the stage refilled below was consumed at ks-1 */
            {
                uint32_t const nxt = ks + IM_STAGES - 1;
                if (nxt < nks) load_slice(tile_base, nxt, nxt % IM_STAGES);
                cp_async_commit();
            }
            uint8_t const* sa = smem + (ks % IM_STAGES) * IM_STAGE_BYTES;
            uint8_t const* sb = sa + IM_BM * IM_BK;
            uint4 fa[4][2], fb[4];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) {
                int const row = wm * 64 + mi * 16 + g;
                fa[mi][0] = *reinterpret_cast<uint4 const*>(sa + row * IM_BK + t * 16);
                fa[mi][1] = *reinterpret_cast<uint4 const*>(sa + (row + 8) * IM_BK + t * 16);
            }
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) fb[ni] = *reinterpret_cast<uint4 const*>(sb + (wn * 32 + ni * 8 + g) * IM_BK + t * 16);
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    imma_16832(acc[mi][ni], fa[mi][0].x, fa[mi][1].x, fa[mi][0].y, fa[mi][1].y, fb[ni].x, fb[ni].y);
                    imma_16832(acc[mi][ni], fa[mi][0].z, fa[mi][1].z, fa[mi][0].w, fa[mi][1].w, fb[ni].z, fb[ni].w);
                }
        }
        cp_async_wait<0>();
        __syncthreads(); /* every warp is done with the stages: the distance tile may overwrite them */

#pragma unroll
        for (int mi = 0; mi < 4; ++mi)
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) {
                int const r0 = wm * 64 + mi * 16 + g, c0 = wn * 32 + ni * 8 + 2 * t;
                float2 lo, hi;
                lo.x = i8_distance<METRIC, SWAP>(acc[mi][ni][0], qa2[r0], vb2[c0], qrn[r0], vrn[c0]);
                lo.y = i8_distance<METRIC, SWAP>(acc[mi][ni][1], qa2[r0], vb2[c0 + 1], qrn[r0], vrn[c0 + 1]);
                hi.x = i8_distance<METRIC, SWAP>(acc[mi][ni][2], qa2[r0 + 8], vb2[c0], qrn[r0 + 8], vrn[c0]);
                hi.y = i8_distance<METRIC, SWAP>(acc[mi][ni][3], qa2[r0 + 8], vb2[c0 + 1], qrn[r0 + 8], vrn[c0 + 1]);
                *reinterpret_cast<float2*>(dist + r0 * IM_DIST_STRIDE + c0) = lo;
                *reinterpret_cast<float2*>(dist + (r0 + 8) * IM_DIST_STRIDE + c0) = hi;
            }
        __syncthreads();

        /* each warp owns 16 query rows: threshold, then the rare sorted insert into the list in global memory */
        for (int rr = 0; rr < 16; ++rr) {
            int const row = warp * 16 + rr;
            uint32_t const qi = q0 + (uint32_t)row;
            if (qi >= (LISTED ? q_end : a.nq)) break; /* warp-uniform */
            uint32_t size = rsize[row];
            float worst = rworst[row];
            size_t const list = ((size_t)qi * a.segments + blockIdx.y) * a.k;
            /* lane l looks at columns 4l..4l+3 in one LDS.128; in the common case nothing passes and one ballot
             * settles the whole row */
            float4 const d4 = *reinterpret_cast<float4 const*>(dist + row * IM_DIST_STRIDE + lane * 4);
            uint32_t const usable4 = (vmask[lane >> 3] >> ((lane & 7) * 4)) & 0xFu;
            float const dv[4] = {d4.x, d4.y, d4.z, d4.w};
            uint32_t pass = 0;
#pragma unroll
            for (int c = 0; c < 4; ++c) pass |= (((usable4 >> c) & 1u) && (size < a.k || !(dv[c] > worst))) ? (1u << c) : 0u;
            if (__ballot_sync(0xffffffffu, pass != 0)) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    uint32_t todo = __ballot_sync(0xffffffffu, (pass >> c) & 1u);
                    while (todo) {
                        int const src_lane = __ffs(todo) - 1;
                        todo &= todo - 1;
                        float const cd = __shfl_sync(0xffffffffu, dv[c], src_lane);
                        uint32_t cs = tile_base + (uint32_t)(src_lane * 4 + c);
                        if constexpr (LISTED) cs = listed_slots[cs];
                        if (size < a.k || !(cd > worst)) {
                            top_insert_global_keyed(a.part_d + list, a.part_s + list, size, a.k, cd, cs, lane);
                            if (size == a.k) worst = reinterpret_cast<float volatile*>(a.part_d)[list + a.k - 1];
                        }
                    }
                }
            }
            if (lane == 0) { rsize[row] = size; rworst[row] = worst; }
        }
        __syncthreads(); /* the distance tile is free again: the next prologue may refill the stages */
    }

    if (tid < IM_BM && q0 + tid < (LISTED ? q_end : a.nq)) a.part_n[(size_t)(q0 + tid) * a.segments + blockIdx.y] = rsize[tid];
}

size_t exact_imma_smem_bytes() { return IM_PIPE_BYTES + (IM_BM + IM_BN) * 8 + IM_BM * 8 + 16; }
int exact_imma_tile_queries() { return IM_BM; }
int exact_imma_tile_vectors() { return IM_BN; }

cudaError_t exact_imma_self_dots(uint8_t const* rows, uint64_t stride, uint32_t chunks16, uint32_t count, int* out, cudaStream_t stream) {
    if (!count) return cudaSuccess;
    i8_self_dot_kernel<<<(count * 32u + 255u) / 256u, 256, 0, stream>>>(rows, stride, chunks16, count, out);
    return cudaGetLastError();
}

cudaError_t exact_imma_listed_self_dots(uint8_t const* vectors, uint64_t stride, uint32_t chunks16, uint32_t const* rows, uint32_t count,
                                        int* out, cudaStream_t stream) {
    if (!count) return cudaSuccess;
    i8_listed_self_dot_kernel<<<(unsigned)(((uint64_t)count * 32u + 255u) / 256u), 256, 0, stream>>>(vectors, stride, chunks16, rows, count,
                                                                                                      out);
    return cudaGetLastError();
}

template <uint32_t METRIC> static cudaError_t imma_launch_t(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream) {
    size_t const smem = exact_imma_smem_bytes();
    if (swap) {
        cudaError_t e = cudaFuncSetAttribute(exact_imma_kernel<METRIC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_imma_kernel<METRIC, true><<<grid, IM_THREADS, smem, stream>>>(ix, a);
    } else {
        cudaError_t e = cudaFuncSetAttribute(exact_imma_kernel<METRIC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_imma_kernel<METRIC, false><<<grid, IM_THREADS, smem, stream>>>(ix, a);
    }
    return cudaGetLastError();
}

template <uint32_t METRIC> static cudaError_t imma_listed_launch_t(exact_listed_args_t const& a, device_index_t const& ix, dim3 grid,
                                                                 cudaStream_t stream) {
    size_t const smem = exact_imma_smem_bytes();
    cudaError_t e = cudaFuncSetAttribute(exact_imma_kernel<METRIC, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    exact_imma_kernel<METRIC, false, true><<<grid, IM_THREADS, smem, stream>>>(ix, a);
    return cudaGetLastError();
}

cudaError_t exact_imma_listed_launch(device_index_t const& ix, exact_listed_args_t const& a, dim3 grid, cudaStream_t stream) {
    switch (ix.metric) {
    case METRIC_IP: return imma_listed_launch_t<METRIC_IP>(a, ix, grid, stream);
    case METRIC_L2SQ: return imma_listed_launch_t<METRIC_L2SQ>(a, ix, grid, stream);
    case METRIC_COS: return imma_listed_launch_t<METRIC_COS>(a, ix, grid, stream);
    default: return cudaErrorInvalidValue;
    }
}

cudaError_t exact_imma_launch(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream) {
    switch (ix.metric) {
    case METRIC_IP: return imma_launch_t<METRIC_IP>(ix, a, swap, grid, stream);
    case METRIC_L2SQ: return imma_launch_t<METRIC_L2SQ>(ix, a, swap, grid, stream);
    case METRIC_COS: return imma_launch_t<METRIC_COS>(ix, a, swap, grid, stream);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace usearch_b200
