// dfb_gl.cu -- GroupedLinearEinsum (DeepFilterNet/df/modules.py:741-780) on the BF16 tensor pipe.
//
//   Y[m, g*Hg + n] = act( sum_i X[m, g*Ig + i] * W[g][i][n] ) * oscale + ooffset + R[m, g*Hg + n]
//
// at fp32-level accuracy (BF16x3: both operands as BF16 hi/lo planes, products hi*hi + lo*hi + hi*lo, fp32
// accumulation).  The block-diagonal weight is NOT expanded to a dense matrix: every group is its own small product
// (16-column chunks of Hg padded to a multiple of 16, K = Ig in steps of 16), so a K step only multiplies the columns
// of the group it belongs to.
//
// Persistent CTA = (group slice, row-tile group).  Its weight slice (gpc groups, <= 100 KB as BF16 hi | lo) is fetched
// once with two bulk copies and stays in shared memory as the B operand (K-major, 8 x 16 B core matrices -- the image is
// laid out on the host, weights.py gl_bx_image).  The X planes [M][K] (written by the producing kernel's epilogue)
// stream through a TMA ring of [128 rows x 64 k] hi + lo boxes (128-byte swizzle) as the A operand.  A K step of 16
// never straddles a box or a group (Ig % 16 == 0, slice start % 64 == 0).
//   warps 0-7 : rows [16 w, +16) of every row tile, all gpc * Hgp <= 256 columns of the slice (ldmatrix + mma.sync,
//               accumulators in registers), then activation / scale / residual -> fp32 and/or BF16 hi/lo plane stores
//   warp 8    : TMA producer
// Staged fp32 output (when y is written and shared memory holds a [128][gpc * Hg] fp32 tile next to a ring of >= 2
// stages): each warp owns the 16 rows of the tile it computes.  The producer loads the warp's residual rows (if any) with
// a TMA box onto the warp's own mbarrier, issued after the tile's X boxes; the warp adds them from shared memory, writes
// the result over them (padded columns dropped, so the slice's gpc * Hg columns are contiguous) and lane 0 stores the 16
// rows with one TMA tensor store (rows >= M are clipped).  Before the rows are overwritten again (by the next residual
// box, or by the warp itself), lane 0 waits for the store to have read them.  The epilogue thus never waits on DRAM, and
// its stores drain while the warp runs the next tile's MMAs.  df_out adds its residual in place (res == y): that is safe
// because a warp's residual rows are read before the same warp's rows of y are stored, and the other CTAs own other
// columns (slices) or other row tiles.
// Staged planes (stage_p, see launch_gl_bx for the shapes that keep register stores): each warp writes the BF16 hi / lo
// planes of 64 output columns at a time into one of its two [16][64] staging blocks (128-byte swizzle, conflict-free for
// the accumulator fragment) and lane 0 stores the block with one TMA tensor store per plane while the warp fills the other.
#include <cuda.h>
#include <cuda_bf16.h>

#include <map>
#include <mutex>
#include <tuple>

#include "dfb_common.cuh"
#include "dfb_dwpw.cuh"
#include "dfb_ptx.cuh"

namespace dfb {

constexpr int kGxThreads = 288, kGxMaxStages = 6, kGxBoxBytes = 128 * 128 /* 128 rows x 64 bf16 */;
constexpr int kGxMaxChunks = 16;                      // 16-column chunks of the slice (gpc * Hgp <= 256)
constexpr uint32_t kGxPlaneBlockBytes = 4096;         // one staged 64-column plane block: hi | lo, 16 rows x 128 B each
constexpr uint32_t kGxPlaneWarpBytes = 2 * kGxPlaneBlockBytes;   // a warp's two blocks (one filled while the other drains)

struct GlBxParams {
    const unsigned short *w_img;  // [hi | lo][G][Ig/8][Hgp/8][8][8] BF16
    const float *res; int64_t ldr;
    float *y; int64_t ldy;
    unsigned short *y_hi, *y_lo; int64_t ldp;
    int M, G, Ig, Hg, Hgp, gpc, act, stages;
    float oscale, ooffset;
    int stage_y;   // fp32 output through the shared staging tile + TMA store (residual, if any, through TMA loads)
    int stage_p;   // BF16 planes through per-warp staging blocks + TMA stores (Hg % 16 == 0, gpc * Hg % 64 == 0)
};

__device__ __forceinline__ float gx_act(float x, int act) {
    if (act == 1) return fmaxf(x, 0.f);
    if (act == 2) return gt_tanh(x);   // 1 - 2 / (1 + e^2x) on the MUFU units (~1e-7 absolute, as in the GRU gates); tanhf made df_out epilogue bound
    return x;
}

// BF16 pair (hi, lo) of row r, column 16 (c % 4) + cc of the warp's 64-column plane block at sp (hi [16][64] | lo [16][64],
// 128-byte swizzle as the TMA store reads it: conflict-free for the 8 rows of a fragment)
__device__ __forceinline__ void gl_stage_planes(uint32_t sp, int c, int r, int cc, float x0, float x1) {
    uint32_t hv, lv;
    bf16x2_split(x0, x1, hv, lv);
    const uint32_t o = sw128_off(r, 2 * (c & 3) + (cc >> 3)) + (uint32_t)(cc & 7) * 2u;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sp + o), "r"(hv) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sp + 2048u + o), "r"(lv) : "memory");
}

// gl_store_chunk with staged planes (p.stage_p): the planes of chunk c go to the warp's staging block sp of the chunk's 64
// columns.  Hg % 16 == 0, so the chunk is slice columns [16 c, +16).  A residual is read from the staging rows st: planes are
// staged without fp32 rows only when there is none.
__device__ __noinline__ void gl_stage_chunk(const GlBxParams &p, int c, uint32_t st, uint32_t sp, float a00, float a01, float a02,
                                            float a03, float a10, float a11, float a12, float a13) {
    const float a[2][4] = {{a00, a01, a02, a03}, {a10, a11, a12, a13}};
    const int lane = threadIdx.x & 31;
    const uint32_t pitch = (uint32_t)(p.gpc * p.Hg) * 4u;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        const int cc = j * 8 + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint32_t sa = st + (uint32_t)((lane >> 2) + 8 * h) * pitch + (uint32_t)(16 * c + cc) * 4u;
            float2 rv = make_float2(0.f, 0.f);
            if (st && p.res) asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(rv.x), "=f"(rv.y) : "r"(sa));
            float2 x;
            x.x = gx_act(a[j][2 * h], p.act) * p.oscale + p.ooffset + rv.x;
            x.y = gx_act(a[j][2 * h + 1], p.act) * p.oscale + p.ooffset + rv.y;
            if (st) sts64(sa, __float_as_uint(x.x), __float_as_uint(x.y));
            gl_stage_planes(sp, c, (lane >> 2) + 8 * h, cc, x.x, x.y);
        }
    }
}

// epilogue of one 16-column chunk c: fragment (n-tile j, half h) = rows mrow + 8 h, columns 2 (lane % 4) + {0, 1} of the n-tile.
// st != 0: the warp's fp32 staging rows [16][gpc * Hg] (holding the residual rows when p.res): y goes there, planes to HBM
__device__ __noinline__ void gl_store_chunk(const GlBxParams &p, int c, int g0, int cpg, int64_t mrow, int lane, uint32_t st,
                                            float a00, float a01, float a02, float a03, float a10, float a11, float a12, float a13) {
    const float a[2][4] = {{a00, a01, a02, a03}, {a10, a11, a12, a13}};
    const int gl = c / cpg;
    if (st) {
        const uint32_t pitch = (uint32_t)(p.gpc * p.Hg) * 4u;
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int n = (c - gl * cpg) * 16 + j * 8 + 2 * (lane & 3);
            if (n >= p.Hg) continue;
            const int lcol = gl * p.Hg + n;   // column inside the slice
            const int64_t col = (int64_t)g0 * p.Hg + lcol;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t sa = st + (uint32_t)((lane >> 2) + 8 * h) * pitch + (uint32_t)lcol * 4u;
                float2 rv = make_float2(0.f, 0.f);
                if (p.res) asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(rv.x), "=f"(rv.y) : "r"(sa));
                float2 x;
                x.x = gx_act(a[j][2 * h], p.act) * p.oscale + p.ooffset + rv.x;
                x.y = gx_act(a[j][2 * h + 1], p.act) * p.oscale + p.ooffset + rv.y;
                sts64(sa, __float_as_uint(x.x), __float_as_uint(x.y));
                const int64_t m = mrow + 8 * h;
                if (p.y_hi && m < p.M) {
                    uint32_t hv, lv;
                    bf16x2_split(x.x, x.y, hv, lv);
                    *reinterpret_cast<uint32_t *>(p.y_hi + m * p.ldp + col) = hv;
                    *reinterpret_cast<uint32_t *>(p.y_lo + m * p.ldp + col) = lv;
                }
            }
        }
        return;
    }
#pragma unroll
    for (int j = 0; j < 2; j++) {
        const int n = (c - gl * cpg) * 16 + j * 8 + 2 * (lane & 3);   // column inside the group
        if (n >= p.Hg) continue;
        const int64_t col = (int64_t)(g0 + gl) * p.Hg + n;
        // residual rows first, both in flight (as load / store pairs the compiler has to assume that res aliases y
        // -- it does for df_out -- and serialises the DRAM round trips)
        float2 rv[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int64_t m = mrow + 8 * h;
            rv[h] = (p.res && m < p.M) ? *reinterpret_cast<const float2 *>(p.res + m * p.ldr + col) : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int64_t m = mrow + 8 * h;
            if (m >= p.M) continue;
            float2 x;
            x.x = gx_act(a[j][2 * h], p.act) * p.oscale + p.ooffset + rv[h].x;
            x.y = gx_act(a[j][2 * h + 1], p.act) * p.oscale + p.ooffset + rv[h].y;
            if (p.y) *reinterpret_cast<float2 *>(p.y + m * p.ldy + col) = x;
            if (p.y_hi) {
                uint32_t hv, lv;
                bf16x2_split(x.x, x.y, hv, lv);
                *reinterpret_cast<uint32_t *>(p.y_hi + m * p.ldp + col) = hv;
                *reinterpret_cast<uint32_t *>(p.y_lo + m * p.ldp + col) = lv;
            }
        }
    }
}

__global__ void __launch_bounds__(kGxThreads, 1)
k_gl_bx(const __grid_constant__ CUtensorMap tmXhi, const __grid_constant__ CUtensorMap tmXlo, const __grid_constant__ CUtensorMap tmY,
        const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmPh, const __grid_constant__ CUtensorMap tmPl,
        const __grid_constant__ GlBxParams p) {
    extern __shared__ __align__(1024) unsigned char gx_smem_raw[];
    const uint32_t sb = (smem_u32(gx_smem_raw) + 1023u) & ~1023u;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slice = blockIdx.x, g0 = slice * p.gpc;
    const int nch = p.gpc * p.Hgp / 16;                    // 16-column chunks of the slice
    const int cpg = p.Hgp / 16;                            // chunks per group
    const int nboxes = p.gpc * p.Ig / 64;                  // 64-wide K boxes per row tile
    const int ntiles = (p.M + 127) / 128;
    const uint32_t gbytes = (uint32_t)p.Ig * p.Hgp * 2;    // one group's block in one plane
    const uint32_t wplane = gbytes * p.gpc;                // the slice in one plane
    const uint32_t lbo = (uint32_t)(p.Hgp / 8) * 128u;     // stride between K-adjacent core matrices of W
    // shared memory map
    const uint32_t s_x = sb;                                             // [stages][hi | lo][16 KB]
    const uint32_t s_w = s_x + (uint32_t)p.stages * 2 * kGxBoxBytes;     // W hi | lo
    const uint32_t ybox = 16u * (uint32_t)(p.gpc * p.Hg) * 4u;           // one warp's staging rows (fp32)
    const uint32_t s_y = s_w + 2 * wplane;                               // [8 warps][16][gpc * Hg] fp32 (stage_y)
    const uint32_t s_p = s_y + (p.stage_y ? 8 * ybox : 0u);              // [8 warps][2 blocks][hi | lo][16][64] BF16 (stage_p)
    const uint32_t s_bar = (s_p + (p.stage_p ? 8u * kGxPlaneWarpBytes : 0u) + 127u) & ~127u;   // full[6] empty[6] wbar rfull[8] rempty[8]
    const uint32_t b_full = s_bar, b_empty = s_bar + 8 * kGxMaxStages, b_w = b_empty + 8 * kGxMaxStages;
    const uint32_t b_rfull = b_w + 8, b_rempty = b_rfull + 8 * 8;
    const bool res_tma = p.stage_y && p.res;
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; s++) { mbar_init_a(b_full + 8 * s, 1); mbar_init_a(b_empty + 8 * s, 8); }
        mbar_init_a(b_w, 1);
        for (int w = 0; w < 8; w++) { mbar_init_a(b_rfull + 8 * w, 1); mbar_init_a(b_rempty + 8 * w, 1); }
        fence_barrier_init();
        // the weight slice: two bulk copies (hi plane, lo plane)
        mbar_expect_tx_a(b_w, 2 * wplane);
        const unsigned char *src = reinterpret_cast<const unsigned char *>(p.w_img);
        bulk_load(s_w, src + (size_t)g0 * gbytes, wplane, b_w);
        bulk_load(s_w + wplane, src + (size_t)p.G * gbytes + (size_t)g0 * gbytes, wplane, b_w);
    }
    __syncthreads();
    if (warp == 8) {
        // ===== TMA producer
        if (lane == 0) {
            tma_prefetch_desc(&tmXhi); tma_prefetch_desc(&tmXlo);
            if (res_tma) tma_prefetch_desc(&tmR);
            const int col0 = g0 * p.Ig;
            int it = 0, ti = 0;
            for (int tile = blockIdx.y; tile < ntiles; tile += gridDim.y, ti++) {
                for (int b = 0; b < nboxes; b++, it++) {
                    const int s = it % p.stages, n = it / p.stages;
                    if (n > 0) mbar_wait_a(b_empty + 8 * s, (uint32_t)((n - 1) & 1));
                    mbar_expect_tx_a(b_full + 8 * s, 2 * kGxBoxBytes);
                    const uint32_t dst = s_x + (uint32_t)s * 2 * kGxBoxBytes;
                    asm volatile(
                        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                        ::"r"(dst), "l"((uint64_t)&tmXhi), "r"(col0 + b * 64), "r"(tile * 128), "r"(b_full + 8 * s) : "memory");
                    asm volatile(
                        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                        ::"r"(dst + kGxBoxBytes), "l"((uint64_t)&tmXlo), "r"(col0 + b * 64), "r"(tile * 128), "r"(b_full + 8 * s) : "memory");
                }
                // the tile's residual rows, one box per warp, once that warp's store of its previous tile has read them out
                // (after the X boxes: a warp's epilogue of tile ti - 1 needs nothing issued here)
                for (int w = 0; res_tma && w < 8; w++) {
                    if (ti > 0) mbar_wait_a(b_rempty + 8 * w, (uint32_t)((ti - 1) & 1));
                    mbar_expect_tx_a(b_rfull + 8 * w, ybox);
                    asm volatile(
                        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                        ::"r"(s_y + (uint32_t)w * ybox), "l"((uint64_t)&tmR), "r"(g0 * p.Hg), "r"(tile * 128 + 16 * w), "r"(b_rfull + 8 * w)
                        : "memory");
                }
            }
        }
        return;
    }
    // ===== consumers: D[rows 16 w .. +16][chunk c] for every chunk of the slice
    const int mat = lane >> 3, rr = lane & 7;
    mbar_wait_a(b_w, 0);
    const uint32_t st = p.stage_y ? s_y + (uint32_t)warp * ybox : 0u;
    const uint32_t spw = p.stage_p ? s_p + (uint32_t)warp * kGxPlaneWarpBytes : 0u;
    int it = 0, ti = 0;
    for (int tile = blockIdx.y; tile < ntiles; tile += gridDim.y, ti++) {
        float acc[kGxMaxChunks][2][4];
#pragma unroll
        for (int c = 0; c < kGxMaxChunks; c++)
#pragma unroll
            for (int e = 0; e < 8; e++) acc[c][e >> 2][e & 3] = 0.f;
        for (int b = 0; b < nboxes; b++, it++) {
            const int s = it % p.stages, n = it / p.stages;
            mbar_wait_a(b_full + 8 * s, (uint32_t)(n & 1));
            const uint32_t xs = s_x + (uint32_t)s * 2 * kGxBoxBytes;
            // (not unrolled: with the chunk loop below unrolled inside four K steps the body grew past ptxas's unroll limit and
            // the accumulators were demoted to local memory)
#pragma unroll 1
            for (int k = 0; k < 4; k++) {  // K step 16 = 32 bytes inside the 128-byte swizzle row of X
                const int col = b * 64 + k * 16;
                const int gl = col / p.Ig, kk = (col - gl * p.Ig) >> 4;
                uint32_t ah[4], al[4];
                const int r = warp * 16 + rr + ((mat & 1) << 3);
                ldsm_x4(xs + sw128_off(r, 2 * k + (mat >> 1)), ah);
                ldsm_x4(xs + kGxBoxBytes + sw128_off(r, 2 * k + (mat >> 1)), al);
                // W core matrix (k core matrix 2 kk + {0, 1}, column group) of group gl, row = column inside the group
                const uint32_t wa = s_w + (uint32_t)gl * gbytes + (uint32_t)(2 * kk + (mat & 1)) * lbo + (uint32_t)rr * 16u;
#pragma unroll
                for (int c = 0; c < kGxMaxChunks; c++) {
                    const int cg = c - gl * cpg;   // chunk inside group gl
                    if (c >= nch || cg < 0 || cg >= cpg) continue;
                    const uint32_t o = wa + (uint32_t)(2 * cg + (mat >> 1)) * 128u;   // matrices: columns 0-7 | 8-15 of the chunk
                    uint32_t bh[4], bl[4];
                    ldsm_x4(o, bh);
                    ldsm_x4(o + wplane, bl);
                    mma_bf16x3(acc[c][0], ah, al, bh[0], bh[1], bl[0], bl[1]);
                    mma_bf16x3(acc[c][1], ah, al, bh[2], bh[3], bl[2], bl[3]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive_a(b_empty + 8 * s);   // ring slot read
        }
        // ---- epilogue: one out-of-line call per chunk, so that this loop stays unrolled and every accumulator index constant
        //      (as one inline loop ptxas re-rolled it and moved the accumulators to local memory)
        //      Staged planes: chunks 4 b .. 4 b + 3 are the slice's plane columns [64 b, +64), staged in the warp's block b % 2
        //      once the store of block b - 2 has read it (an odd block count drains at the end of the tile).
        const int64_t mrow = (int64_t)tile * 128 + warp * 16 + (lane >> 2);
        if (res_tma) mbar_wait_a(b_rfull + 8 * warp, (uint32_t)(ti & 1));
#pragma unroll
        for (int c = 0; c < kGxMaxChunks; c++) {
            if (c >= nch) continue;
            const uint32_t sp = spw ? spw + (uint32_t)((c >> 2) & 1) * kGxPlaneBlockBytes : 0u;
            if (sp) {
                if ((c & 3) == 0) {
                    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    __syncwarp();
                }
            }
            if (sp)
                gl_stage_chunk(p, c, st, sp, acc[c][0][0], acc[c][0][1], acc[c][0][2], acc[c][0][3], acc[c][1][0], acc[c][1][1],
                               acc[c][1][2], acc[c][1][3]);
            else
                gl_store_chunk(p, c, g0, cpg, mrow, lane, st, acc[c][0][0], acc[c][0][1], acc[c][0][2], acc[c][0][3], acc[c][1][0],
                               acc[c][1][1], acc[c][1][2], acc[c][1][3]);
            if (sp && (c & 3) == 3) {
                // the block's 16 rows -> both planes (two TMA stores; rows >= M are clipped)
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) {
                    const int col = g0 * p.Hg + 16 * (c - 3), row = tile * 128 + warp * 16;
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];"
                                 ::"l"((uint64_t)&tmPh), "r"(col), "r"(row), "r"(sp) : "memory");
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];"
                                 ::"l"((uint64_t)&tmPl), "r"(col), "r"(row), "r"(sp + 2048u) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    if (c + 1 == nch && (nch & 4)) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                }
            }
        }
        if (st) {
            // the staged rows -> y (one TMA store; the tensor map clips rows >= M), read out before the rows are reused
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];"
                             ::"l"((uint64_t)&tmY), "r"(g0 * p.Hg), "r"(tile * 128 + warp * 16), "r"(st) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                if (res_tma) mbar_arrive_a(b_rempty + 8 * warp);
            }
            __syncwarp();
        }
    }
    // the last plane blocks are read out before the CTA's shared memory goes away
    if (p.stage_p && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// ------------------------------------------------------ df_conv1 -> df_fc_emb, c1 kept on chip ----
//   emb_in[m, cols] = relu( GL( relu( pw( dw_s2(c0[m]) ) + b ) ) ) (+ e3[m])
// (deepfilternet3.py:166-185: df_conv1, then df_fc_emb over the flattened c1).  The chain is local to a row m = b T + t
// (kt = 2: and its previous frame), so one CTA owns a slice of S c1 bins (whole GL groups: S * 64 % Ig == 0) of every
// row tile it visits and c1 never leaves the SM.  Per row tile and bin j of the slice, each consumer warp
//   1. forms the depthwise result of its 16 rows right in mma.sync A-fragment layout from the three c0 bins 2j-1 .. 2j+1
//      (fp32 TMA boxes in a ring) and splits it into BF16 hi / lo (BF16x3),
//   2. multiplies it by the 1x1 weight (the df_conv1.pw_sw image in shared memory, ldmatrix),
//   3. turns the accumulators into c1 = relu(acc + b) split into hi / lo -- the accumulator fragments of n-tiles 2k, 2k + 1
//      are the A fragment of K step k of the grouped linear, so c1 stays in registers --
//   4. multiplies that by the slice's GL weights (the df_fc_emb.gl_bx image, resident) into the GL accumulators.
// The arithmetic and its order are those of k_dwpw_bx<DW_S2> followed by k_gl_bx, so the output bits are the same.
//   warps 0-7: rows [16 w, +16) of the tile; warp 8: TMA producer.  A tile is 128 rows of c0 starting KT - 1 rows before
//   its first output row (kt = 2: box row 0 is the halo frame of box row 1), so it produces RT = 128 - (KT - 1) rows.
// Slices of one row tile are adjacent in launch order: the edge bin 2 j0 - 1 that two slices share comes from L2.
constexpr int kDeThreads = 288, kDeMaxStages = 6, kDeMaxChunks = 4;
constexpr uint32_t kDeBin = 32768;   // one c0 bin of a tile: 128 rows x 64 fp32 as two [128][32] swizzled boxes

struct DfEmbParams {
    const float *dw;      // df_conv1 depthwise taps [kt][3][64]
    const float *bias;    // [64]
    const float *pw_sw;   // df_conv1.pw_sw: [hi | lo] x [64 n][64 k] BF16, 128B-swizzled rows
    const unsigned short *w_img;  // df_fc_emb.gl_bx: [hi | lo][G][Ig/8][Hgp/8][8][8] BF16
    const float *res; int64_t ldr;             // e3 or null
    unsigned short *y_hi, *y_lo; int64_t ldp;  // emb_in planes (pre-offset to the first output column)
    int M, T, G, Ig, Hg, Hgp, S, stages;
    float oscale, ooffset;
    const int64_t *first;  // kt = 2, streaming slots: first frame of each stream (stream_first), or null
    int64_t w0;
};

template <int KT>
__global__ void __launch_bounds__(kDeThreads, 1)
k_dwpw_gl(const __grid_constant__ CUtensorMap tmC0, const __grid_constant__ DfEmbParams p) {
    extern __shared__ __align__(1024) unsigned char de_smem_raw[];
    const uint32_t sb = (smem_u32(de_smem_raw) + 1023u) & ~1023u;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int RT = 128 - (KT - 1);
    const int ntiles = (p.M + RT - 1) / RT;
    const int j0 = blockIdx.x * p.S;                          // c1 bins [j0, j0 + S)
    const int f_lo = j0 > 0 ? 2 * j0 - 1 : 0, f_hi = 2 * (j0 + p.S);   // c0 bins [f_lo, f_hi) of every tile
    const int gps = p.S * kCh / p.Ig, cpg = p.Hgp / 16, nch = gps * cpg;
    const int g0 = j0 * kCh / p.Ig;                           // first GL group of the slice
    const uint32_t gbytes = (uint32_t)p.Ig * p.Hgp * 2;       // one group's block in one plane
    const uint32_t wplane = gbytes * gps;
    const uint32_t lbo = (uint32_t)(p.Hgp / 8) * 128u;
    // shared memory map
    const uint32_t s_c0 = sb;                                          // [stages][32 KB]
    const uint32_t s_pw = s_c0 + (uint32_t)p.stages * kDeBin;          // 16 KB (1024-aligned)
    const uint32_t s_w = s_pw + 2u * kCh * 128u;                       // GL weights hi | lo
    const uint32_t s_bias = s_w + 2 * wplane;                          // [64]
    const uint32_t s_dw = s_bias + 256u;                               // depthwise taps [KT][3][64]
    const uint32_t s_bar = (s_dw + KT * 3 * kCh * 4u + 127u) & ~127u;
    const uint32_t b_full = s_bar, b_empty = s_bar + 8 * kDeMaxStages, b_w = b_empty + 8 * kDeMaxStages;
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; s++) { mbar_init_a(b_full + 8 * s, 1); mbar_init_a(b_empty + 8 * s, 8); }
        mbar_init_a(b_w, 1);
        fence_barrier_init();
        mbar_expect_tx_a(b_w, 2u * kCh * 128u + 2 * wplane);
        bulk_load(s_pw, p.pw_sw, 2u * kCh * 128u, b_w);
        const unsigned char *src = reinterpret_cast<const unsigned char *>(p.w_img);
        bulk_load(s_w, src + (size_t)g0 * gbytes, wplane, b_w);
        bulk_load(s_w + wplane, src + (size_t)p.G * gbytes + (size_t)g0 * gbytes, wplane, b_w);
    }
    if (threadIdx.x < kCh / 4) sts128(s_bias + threadIdx.x * 16, __ldg(reinterpret_cast<const float4 *>(p.bias) + threadIdx.x));
    for (int i = threadIdx.x; i < KT * 3 * kCh / 4; i += kDeThreads) sts128(s_dw + i * 16, __ldg(reinterpret_cast<const float4 *>(p.dw) + i));
    __syncthreads();
    if (warp == 8) {
        // ===== TMA producer: c0 bins f_lo .. f_hi - 1 of every tile, in order
        if (lane == 0) {
            tma_prefetch_desc(&tmC0);
            int it = 0;
            for (int tile = blockIdx.y; tile < ntiles; tile += gridDim.y) {
                const int row0 = tile * RT - (KT - 1);   // may be -1: out-of-bounds rows arrive as zeros
                for (int f = f_lo; f < f_hi; f++, it++) {
                    const int s = it % p.stages, n = it / p.stages;
                    if (n > 0) mbar_wait_a(b_empty + 8 * s, (uint32_t)((n - 1) & 1));
                    mbar_expect_tx_a(b_full + 8 * s, kDeBin);
                    const uint32_t dst = s_c0 + (uint32_t)s * kDeBin;
                    asm volatile(
                        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                        ::"r"(dst), "l"((uint64_t)&tmC0), "r"(f * kCh), "r"(row0), "r"(b_full + 8 * s) : "memory");
                    asm volatile(
                        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                        ::"r"(dst + kDeBin / 2), "l"((uint64_t)&tmC0), "r"(f * kCh + 32), "r"(row0), "r"(b_full + 8 * s) : "memory");
                }
            }
        }
        return;
    }
    // ===== consumers.  Lane (g = lane / 4, q = lane % 4) holds A-fragment elements of rows 16 w + g + 8 rs and channels
    //       16 ks + 8 h + 2 q + {0, 1} (register rs + 2 h of K step ks)
    const int g = lane >> 2, q = lane & 3, mat = lane >> 3, rr = lane & 7;
    mbar_wait_a(b_w, 0);
    int it = 0;   // ring index of the tile's first c0 bin
    for (int tile = blockIdx.y; tile < ntiles; tile += gridDim.y, it += f_hi - f_lo) {
        const int row0 = tile * RT - (KT - 1);
        // taps present per (row half rs, time tap dt): kt = 2 reads zero padding before the stream's first frame
        bool tap_ok[2][KT];
#pragma unroll
        for (int rs = 0; rs < 2; rs++) {
            const int r = warp * 16 + g + 8 * rs, m = row0 + r;
#pragma unroll
            for (int dt = 0; dt < KT; dt++) tap_ok[rs][dt] = true;
            if (KT > 1) {
                const int b = m >= 0 && m < p.M ? m / p.T : 0, t = m - b * p.T;
                const int t_first = stream_first(p.first, b, p.w0);
#pragma unroll
                for (int dt = 0; dt < KT; dt++) tap_ok[rs][dt] = r - (KT - 1) + dt >= 0 && t - (KT - 1 - dt) >= t_first;
            }
        }
        float gacc[kDeMaxChunks][2][4];
#pragma unroll
        for (int c = 0; c < kDeMaxChunks; c++)
#pragma unroll
            for (int e = 0; e < 8; e++) gacc[c][e >> 2][e & 3] = 0.f;
        for (int jj = 0; jj < p.S; jj++) {
            const int j = j0 + jj;
            // ---- 1. depthwise (taps in the order of k_dwpw_bx: time tap, then bins 2j-1, 2j, 2j+1) -> BF16 hi / lo
            uint32_t slot[3];
#pragma unroll
            for (int df = 0; df < 3; df++) {
                const int f = 2 * j - 1 + df;
                const int i = it + (f < f_lo ? 0 : f - f_lo);
                slot[df] = s_c0 + (uint32_t)(i % p.stages) * kDeBin;
                if (f >= f_lo) mbar_wait_a(b_full + 8 * (i % p.stages), (uint32_t)((i / p.stages) & 1));
            }
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int ks = 0; ks < 4; ks++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int ch = 16 * ks + 8 * h + 2 * q;   // box (ch / 32), 16-byte chunk (ch % 32) / 4, float (ch % 4)
                    const uint32_t cbase = (uint32_t)(ch >> 5) * (kDeBin / 2) + (uint32_t)(ch & 3) * 4u;
                    const int chunk = (ch & 31) >> 2;
#pragma unroll
                    for (int rs = 0; rs < 2; rs++) {
                        const int r = warp * 16 + g + 8 * rs;
                        float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                        for (int dt = 0; dt < KT; dt++) {
                            if (!tap_ok[rs][dt]) continue;
                            const int rb = r - (KT - 1) + dt;   // box row of this time tap
                            const uint32_t o = cbase + (uint32_t)rb * 128u + (uint32_t)((chunk ^ (rb & 7)) << 4);
#pragma unroll
                            for (int df = 0; df < 3; df++) {
                                if (df == 0 && j == 0) continue;
                                float2 x;
                                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x.x), "=f"(x.y) : "r"(slot[df] + o));
                                float2 w;
                                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(w.x), "=f"(w.y) : "r"(s_dw + 4u * ((dt * 3 + df) * kCh + ch)));
                                acc.x = fmaf(x.x, w.x, acc.x);
                                acc.y = fmaf(x.y, w.y, acc.y);
                            }
                        }
                        bf16x2_split(acc.x, acc.y, ah[ks][rs + 2 * h], al[ks][rs + 2 * h]);
                    }
                }
            // c0 bins this warp no longer reads: 2j-1 and 2j (2j+1 is the next bin's left tap, unless j is the slice's last)
            __syncwarp();
            if (lane == 0) {
                for (int f = 2 * j - 1; f <= 2 * j + (jj + 1 == p.S ? 1 : 0); f++)
                    if (f >= f_lo) mbar_arrive_a(b_empty + 8 * ((it + f - f_lo) % p.stages));
            }
            // ---- 2. 1x1 conv (order of warp_mma_sw128_k64<1>)
            float acc[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; nt++)
#pragma unroll
                for (int e = 0; e < 4; e++) acc[nt][e] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 4; ks++)
#pragma unroll
                for (int np = 0; np < 4; np++) {
                    const int n = 16 * np + rr + ((mat >> 1) << 3);
                    const uint32_t o = sw128_off(n, 2 * ks + (mat & 1));
                    uint32_t bh[4], bl[4];
                    ldsm_x4(s_pw + o, bh);
                    ldsm_x4(s_pw + 8192 + o, bl);
                    mma_bf16x3(acc[2 * np], ah[ks], al[ks], bh[0], bh[1], bl[0], bl[1]);
                    mma_bf16x3(acc[2 * np + 1], ah[ks], al[ks], bh[2], bh[3], bl[2], bl[3]);
                }
            // ---- 3. c1 = relu(acc + b) -> BF16 hi / lo A fragments of the grouped linear (K step kk = n-tiles 2 kk, 2 kk + 1)
            uint32_t ch_[4][4], cl_[4][4];
#pragma unroll
            for (int nt = 0; nt < 8; nt++) {
                const int c = 8 * nt + 2 * q;
                float b0, b1;
                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b0), "=f"(b1) : "r"(s_bias + 4 * c));
#pragma unroll
                for (int rs = 0; rs < 2; rs++)
                    bf16x2_split(fmaxf(acc[nt][2 * rs] + b0, 0.f), fmaxf(acc[nt][2 * rs + 1] + b1, 0.f), ch_[nt >> 1][rs + 2 * (nt & 1)],
                                 cl_[nt >> 1][rs + 2 * (nt & 1)]);
            }
            // ---- 4. grouped linear, K = this bin's 64 columns in steps of 16 (order of k_gl_bx)
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                const int col = jj * kCh + kk * 16;
                const int gl = col / p.Ig, kq = (col - gl * p.Ig) >> 4;
                const uint32_t wa = s_w + (uint32_t)gl * gbytes + (uint32_t)(2 * kq + (mat & 1)) * lbo + (uint32_t)rr * 16u;
#pragma unroll
                for (int c = 0; c < kDeMaxChunks; c++) {
                    const int cg = c - gl * cpg;
                    if (c >= nch || cg < 0 || cg >= cpg) continue;
                    const uint32_t o = wa + (uint32_t)(2 * cg + (mat >> 1)) * 128u;
                    uint32_t bh[4], bl[4];
                    ldsm_x4(o, bh);
                    ldsm_x4(o + wplane, bl);
                    mma_bf16x3(gacc[c][0], ch_[kk], cl_[kk], bh[0], bh[1], bl[0], bl[1]);
                    mma_bf16x3(gacc[c][1], ch_[kk], cl_[kk], bh[2], bh[3], bl[2], bl[3]);
                }
            }
        }
        // ---- epilogue (formula of gl_store_chunk): rows below the tile's first output row are the previous tile's
        const int64_t mrow = (int64_t)row0 + warp * 16 + g;
        const int64_t mmin = (int64_t)tile * RT;
#pragma unroll
        for (int c = 0; c < kDeMaxChunks; c++) {
            if (c >= nch) continue;
            const int gl = c / cpg;
#pragma unroll
            for (int jh = 0; jh < 2; jh++) {
                const int n = (c - gl * cpg) * 16 + jh * 8 + 2 * q;
                if (n >= p.Hg) continue;
                const int64_t col = (int64_t)(g0 + gl) * p.Hg + n;
                float2 rv[2];
#pragma unroll
                for (int rs = 0; rs < 2; rs++) {
                    const int64_t m = mrow + 8 * rs;
                    rv[rs] = (p.res && m >= mmin && m < p.M) ? *reinterpret_cast<const float2 *>(p.res + m * p.ldr + col) : make_float2(0.f, 0.f);
                }
#pragma unroll
                for (int rs = 0; rs < 2; rs++) {
                    const int64_t m = mrow + 8 * rs;
                    if (m < mmin || m >= p.M) continue;
                    float2 x;
                    x.x = gx_act(gacc[c][jh][2 * rs], 1) * p.oscale + p.ooffset + rv[rs].x;
                    x.y = gx_act(gacc[c][jh][2 * rs + 1], 1) * p.oscale + p.ooffset + rv[rs].y;
                    uint32_t hv, lv;
                    bf16x2_split(x.x, x.y, hv, lv);
                    *reinterpret_cast<uint32_t *>(p.y_hi + m * p.ldp + col) = hv;
                    *reinterpret_cast<uint32_t *>(p.y_lo + m * p.ldp + col) = lv;
                }
            }
        }
    }
}

// fp32 [M][K] (row pitch ldx) -> BF16 hi / lo planes [M][K] (pitch K): fallback producer for inputs whose own
// producer wrote none (ensure_planes in dfb_model.cu)
__global__ void __launch_bounds__(256) k_to_planes(const float *__restrict__ x, int64_t ldx, int64_t M, int K,
                                                   unsigned short *__restrict__ hi, unsigned short *__restrict__ lo) {
    const int64_t n4 = M * (K / 4);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / (K / 4);
        const int k = (int)(i - m * (K / 4)) * 4;
        const float4 v = *reinterpret_cast<const float4 *>(x + m * ldx + k);
        uint32_t h0, l0, h1, l1;
        bf16x2_split(v.x, v.y, h0, l0);
        bf16x2_split(v.z, v.w, h1, l1);
        *reinterpret_cast<uint2 *>(hi + m * K + k) = make_uint2(h0, h1);
        *reinterpret_cast<uint2 *>(lo + m * K + k) = make_uint2(l0, l1);
    }
}

// ------------------------------------------------------------------------------- host side ----
typedef CUresult (*PFN_encodeTiled_gl)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                       const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                       CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Tensor maps are cached per (device, base, rows, cols, pitch): the arena hands out the same addresses call after call,
// so steady-state launches do not re-encode.
int cached_map_bf16(CUtensorMap *out, const void *base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, int64_t, int64_t, int64_t, int>, CUtensorMap> cache;
    static PFN_encodeTiled_gl enc = nullptr;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    auto key = std::make_tuple(dev, base, rows, cols, ld, box_rows);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return DFB_OK; }
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return fail(DFB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
        enc = (PFN_encodeTiled_gl)fp;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(DFB_ERR_CUDA, "cuTensorMapEncodeTiled (bf16) failed (%d)", (int)r);
    if (cache.size() > 4096) cache.clear();
    cache[key] = m;
    *out = m;
    return DFB_OK;
}

// 2-D fp32 row-major [rows][cols] (row pitch ld floats), box = [box_rows][32 floats = 128 B], 128-byte swizzle
int cached_map_f32_sw128(CUtensorMap *out, const void *base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, int64_t, int64_t, int64_t, int>, CUtensorMap> cache;
    static PFN_encodeTiled_gl enc = nullptr;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    auto key = std::make_tuple(dev, base, rows, cols, ld, box_rows);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return DFB_OK; }
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return fail(DFB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
        enc = (PFN_encodeTiled_gl)fp;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {32u, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(DFB_ERR_CUDA, "cuTensorMapEncodeTiled (fp32) failed (%d)", (int)r);
    if (cache.size() > 4096) cache.clear();
    cache[key] = m;
    *out = m;
    return DFB_OK;
}

// 2-D fp32 row-major [rows][cols] (row pitch ld floats), box = [box_rows][box_cols], no swizzle: the staged epilogue of
// k_gl_bx (residual loads, y stores)
static int cached_map_f32_rows(CUtensorMap *out, const void *base, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows) {
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, int64_t, int64_t, int64_t, int, int>, CUtensorMap> cache;
    static PFN_encodeTiled_gl enc = nullptr;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    auto key = std::make_tuple(dev, base, rows, cols, ld, box_cols, box_rows);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return DFB_OK; }
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return fail(DFB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
        enc = (PFN_encodeTiled_gl)fp;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(DFB_ERR_CUDA, "cuTensorMapEncodeTiled (fp32 rows) failed (%d)", (int)r);
    if (cache.size() > 4096) cache.clear();
    cache[key] = m;
    *out = m;
    return DFB_OK;
}

int launch_to_planes(cudaStream_t s, const float *x, int64_t ldx, int64_t M, int K, unsigned short *hi, unsigned short *lo) {
    if (K % 4 || ldx % 4) return fail(DFB_ERR_UNSUPPORTED, "to_planes: K = %d", K);
    int dev = 0, sms = 0;
    DFB_CUDA(cudaGetDevice(&dev));
    DFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    DFB_PROF("k_to_planes", s);
    k_to_planes<<<sms * 8, 256, 0, s>>>(x, ldx, M, K, hi, lo);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

// Geometry of the tensor-core grouped linear for (G, Ig, Hg); returns false when the shape is outside the kernel.
bool gl_bx_geometry(int G, int Ig, int Hg, int *gpc_out, int *hgp_out, int *stages_out) {
    if (Ig % 16 || Hg % 4 || G < 1) return false;
    const int Hgp = (Hg + 15) / 16 * 16;
    if (Hgp > 256) return false;
    int best = 0;
    for (int gpc = 1; gpc <= G; gpc++) {
        if (G % gpc) continue;
        if (gpc * Hgp > 256 || (gpc * Hgp) % 32) continue;
        if ((gpc * Ig) % 64) continue;
        if ((size_t)gpc * Ig * Hgp * 4 > 100 * 1024) continue;
        best = gpc;
    }
    if (!best) return false;
    const int w = best * Ig * Hgp * 4;
    int stages = (227 * 1024 - 2048 - w - 256) / (2 * kGxBoxBytes);
    if (stages > kGxMaxStages) stages = kGxMaxStages;
    if (stages < 2) return false;
    *gpc_out = best; *hgp_out = Hgp; *stages_out = stages;
    return true;
}

// Y = act(GL(X)) ... with X given as BF16 planes [M][K = G * Ig] (pitch ldx elements) and the host-packed weight image.
int launch_gl_bx(cudaStream_t s, const unsigned short *x_hi, const unsigned short *x_lo, int64_t ldx, const float *w_img,
                 const float *res, int64_t ldr, float *y, int64_t ldy, unsigned short *y_hi, unsigned short *y_lo, int64_t ldp,
                 int64_t M, int G, int Ig, int Hg, int act, float oscale, float ooffset) {
    int gpc = 0, Hgp = 0, stages = 0;
    if (!gl_bx_geometry(G, Ig, Hg, &gpc, &Hgp, &stages) || M <= 0 || M > 0x7fffffff || (ldx % 8) || ((uintptr_t)x_hi & 15) ||
        ((uintptr_t)x_lo & 15) || (y && ((ldy % 4) || ((uintptr_t)y & 15))) || (res && ((ldr % 4) || ((uintptr_t)res & 15))) ||
        (y_hi && ((ldp % 4) || ((uintptr_t)y_hi & 7) || ((uintptr_t)y_lo & 7))))
        return DFB_ERR_UNSUPPORTED;
    CUtensorMap mh, ml;
    int rc;
    if ((rc = cached_map_bf16(&mh, x_hi, M, (int64_t)G * Ig, ldx, 128)) || (rc = cached_map_bf16(&ml, x_lo, M, (int64_t)G * Ig, ldx, 128)))
        return rc;
    // staged outputs come out of the ring, which keeps >= 2 stages.  fp32: the [128][gpc * Hg] staging tile.  Planes: two
    // [16][64] hi | lo blocks per warp, stored as 64-column TMA boxes; they stay stored from registers when
    //   - Hg % 16 or gpc * Hg % 64 (a 16-column chunk would straddle a group or the slice would end inside a block),
    //   - ldp % 8, or a plane base not 16-byte aligned (TMA needs 16-byte global strides and addresses),
    //   - y is written but not staged, or a residual is added without y (those rows come from registers too), or
    //   - the ring would drop below 2 stages (e.g. DeepFilterNet3 enc.emb_gru.out: weights + fp32 tile leave room for 2).
    const int wbytes = gpc * Ig * Hgp * 4, ybytes = 128 * gpc * Hg * 4, pbytes = 8 * (int)kGxPlaneWarpBytes;
    auto ring = [&](int staged) {
        const int s = (227 * 1024 - 2048 - wbytes - staged - 256) / (2 * kGxBoxBytes);
        return s > kGxMaxStages ? kGxMaxStages : s;
    };
    const bool stage_y = y && ring(ybytes) >= 2;
    const bool stage_p = y_hi && Hg % 16 == 0 && (gpc * Hg) % 64 == 0 && ldp % 8 == 0 && !((uintptr_t)y_hi & 15) &&
                         !((uintptr_t)y_lo & 15) && (y ? stage_y : !res) && ring((stage_y ? ybytes : 0) + pbytes) >= 2;
    CUtensorMap my = mh, mr = mh, mph = mh, mpl = mh;   // (unused copies when not staged / no residual)
    if (stage_y) {
        if ((rc = cached_map_f32_rows(&my, y, M, (int64_t)G * Hg, ldy, gpc * Hg, 16))) return rc;
        if (res && (rc = cached_map_f32_rows(&mr, res, M, (int64_t)G * Hg, ldr, gpc * Hg, 16))) return rc;
    }
    if (stage_p && ((rc = cached_map_bf16(&mph, y_hi, M, (int64_t)G * Hg, ldp, 16)) || (rc = cached_map_bf16(&mpl, y_lo, M, (int64_t)G * Hg, ldp, 16))))
        return rc;
    const int staged = (stage_y ? ybytes : 0) + (stage_p ? pbytes : 0);
    if (staged) stages = ring(staged);
    GlBxParams p{reinterpret_cast<const unsigned short *>(w_img), res, ldr, y, ldy, y_hi, y_lo, ldp,
                 (int)M, G, Ig, Hg, Hgp, gpc, act, stages, oscale, ooffset, stage_y ? 1 : 0, stage_p ? 1 : 0};
    const int smem = 1024 + stages * 2 * kGxBoxBytes + wbytes + staged + 128 + 256;
    static PerDeviceOnce attr_once;
    if (auto once_guard = attr_once.first())
        DFB_CUDA(cudaFuncSetAttribute(k_gl_bx, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    int dev = 0, sms = 0;
    DFB_CUDA(cudaGetDevice(&dev));
    DFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int slices = G / gpc, ntiles = (int)((M + 127) / 128);
    int groups = sms / slices;
    if (groups < 1) groups = 1;
    if (groups > ntiles) groups = ntiles;
    DFB_PROF("k_gl_bx", s);
    k_gl_bx<<<dim3((unsigned)slices, (unsigned)groups), kGxThreads, smem, s>>>(mh, ml, my, mr, mph, mpl, p);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

}  // namespace dfb

// Debug aid (bench_gl.py, tests/test_gpu_gl_bx.py): one k_gl_bx launch on caller-given device pointers
extern "C" int dfb_debug_gl_bx(const void *x_hi, const void *x_lo, int64_t ldx, const float *w_img, const float *res, int64_t ldr,
                               float *y, int64_t ldy, void *y_hi, void *y_lo, int64_t ldp, int64_t M, int G, int Ig, int Hg,
                               int act, float oscale, float ooffset, void *stream) {
    if (!x_hi || !x_lo || !w_img || (!y && !y_hi) || (!y_hi != !y_lo)) return dfb::fail(DFB_ERR_INVALID, "gl_bx: null argument");
    const int r = dfb::launch_gl_bx((cudaStream_t)stream, (const unsigned short *)x_hi, (const unsigned short *)x_lo, ldx, w_img, res,
                                    ldr, y, ldy, (unsigned short *)y_hi, (unsigned short *)y_lo, ldp, M, G, Ig, Hg, act, oscale, ooffset);
    if (r == DFB_ERR_UNSUPPORTED) return dfb::fail(r, "gl_bx: shape G %d Ig %d Hg %d or pointer alignment not built", G, Ig, Hg);
    return r;
}

namespace dfb {

// Slice width S (c1 bins per CTA: the fewest that hold whole GL groups) and ring depth of k_dwpw_gl for df_fc_emb = (G, Ig,
// Hg) over Fd / 2 c1 bins; false when the shape is outside the kernel (the caller keeps df_conv1 and df_fc_emb apart).
bool df_emb_geometry(int Fd, int G, int Ig, int Hg, int kt, int *s_out, int *stages_out) {
    if ((kt != 1 && kt != 2) || Fd % 2 || Ig % 16 || Hg % 4 || G < 1 || G * Ig != Fd / 2 * kCh) return false;
    int S = 1;
    while ((S * kCh) % Ig) S++;
    const int Hgp = (Hg + 15) / 16 * 16;
    if ((Fd / 2) % S || (S * kCh / Ig) * (Hgp / 16) > kDeMaxChunks) return false;
    const int fixed = 1024 + 2 * kCh * 128 + S * kCh * Hgp * 4 + 256 + kt * 3 * kCh * 4 + 128 + 2 * 8 * kDeMaxStages + 8;
    int stages = (227 * 1024 - fixed) / (int)kDeBin;
    if (stages > kDeMaxStages) stages = kDeMaxStages;
    if (stages < 3) return false;   // bins 2j-1 .. 2j+1 are in use at once
    *s_out = S; *stages_out = stages;
    return true;
}

// emb_in planes (y_hi / y_lo, pitch ldp, pre-offset to the first column) = relu(df_fc_emb(df_conv1(c0))) (+ res) over
// M = B * T rows of c0 [M][Fd][64]
int launch_df_emb(cudaStream_t s, const float *c0, int64_t M, int T, int Fd, int kt, const float *dw, const float *bias,
                  const float *pw_sw, const float *w_img, int G, int Ig, int Hg, const float *res, int64_t ldr,
                  unsigned short *y_hi, unsigned short *y_lo, int64_t ldp, const int64_t *first, int64_t w0) {
    int S = 0, stages = 0;
    if (!df_emb_geometry(Fd, G, Ig, Hg, kt, &S, &stages) || M <= 0 || M > 0x7fffffff - 256 || T <= 0 || M % T ||
        (res && ((ldr % 2) || ((uintptr_t)res & 7))) || (ldp % 2) || ((uintptr_t)y_hi & 3) || ((uintptr_t)y_lo & 3) ||
        ((uintptr_t)c0 & 15) || ((uintptr_t)w_img & 15) || ((uintptr_t)pw_sw & 15))
        return fail(DFB_ERR_UNSUPPORTED, "df_conv1 + df_fc_emb kernel: shape G %d Ig %d Hg %d kt %d", G, Ig, Hg, kt);
    CUtensorMap mc;
    int rc;
    if ((rc = cached_map_f32_sw128(&mc, c0, M, (int64_t)Fd * kCh, (int64_t)Fd * kCh, 128))) return rc;
    const int Hgp = (Hg + 15) / 16 * 16;
    DfEmbParams p{dw, bias, pw_sw, reinterpret_cast<const unsigned short *>(w_img), res, ldr, y_hi, y_lo, ldp,
                  (int)M, T, G, Ig, Hg, Hgp, S, stages, 1.f, 0.f, first, w0};
    const int smem = 1024 + stages * (int)kDeBin + 2 * kCh * 128 + S * kCh * Hgp * 4 + 256 + kt * 3 * kCh * 4 + 128 + 2 * 8 * kDeMaxStages + 8;
    static PerDeviceOnce attr_once;
    if (auto once_guard = attr_once.first()) {
        DFB_CUDA(cudaFuncSetAttribute(k_dwpw_gl<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        DFB_CUDA(cudaFuncSetAttribute(k_dwpw_gl<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    int dev = 0, sms = 0;
    DFB_CUDA(cudaGetDevice(&dev));
    DFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int slices = Fd / 2 / S, rt = 128 - (kt - 1);
    const int ntiles = (int)((M + rt - 1) / rt);
    int groups = sms / slices;
    if (groups < 1) groups = 1;
    if (groups > ntiles) groups = ntiles;
    DFB_PROF("k_dwpw_gl", s);
    if (kt == 1) k_dwpw_gl<1><<<dim3((unsigned)slices, (unsigned)groups), kDeThreads, smem, s>>>(mc, p);
    else k_dwpw_gl<2><<<dim3((unsigned)slices, (unsigned)groups), kDeThreads, smem, s>>>(mc, p);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

}  // namespace dfb
