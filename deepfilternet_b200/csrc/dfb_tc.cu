// dfb_tc.cu -- tensor-core (BF16 mma.sync) kernels for the dense contractions of the path.
//
//   k_gemm_bf16x3: GRU input projections W_ih x + b_ih (torch.nn.GRU inside SqueezedGRU[_S], modules.py:684,723)
//   k_dwpw_bx:     fused depthwise (+pathway) -> 1x1 conv -> ReLU blocks (Conv2dNormAct / ConvTranspose2dNormAct)
//   k_df_convp_tc: the DF pathway conv (channel contraction on the tensor pipe, shifted sums in the epilogue)
//   k_gru_tc:      the GRU recurrence W_hh h with the weights resident on chip
// All of them reach fp32-level accuracy on the BF16 tensor pipe by splitting both operands into BF16 hi + lo planes
// (x = hi + lo to ~2^-17) and issuing hi*hi + lo*hi + hi*lo with fp32 accumulation in registers.
#include <cooperative_groups.h>
#include <atomic>
#include <map>
#include <mutex>
#include <cuda.h>
#include <cuda_bf16.h>

#include "dfb_common.cuh"
#include "dfb_dwpw.cuh"
#include "dfb_ptx.cuh"

namespace dfb {

// ------------------------------------------------------------- BF16x3 GEMM (projections) ----
// Y[M,N] = X[M,K] . W[N,K]^T + bias with fp32-level accuracy on the BF16 tensor pipe: both operands are stored as BF16
// hi/lo planes (x = hi + lo to ~2^-17; X planes written by the producing kernel's epilogue, W planes split on the host)
// and every product is hi*hi + lo*hi + hi*lo with fp32 accumulation.
// One CTA = a 128 x 128 output tile.  Warp 8 is the TMA producer: per 64-wide K block it loads the X and W boxes
// ([128 rows][64 k], hi + lo, 128-byte swizzle, 64 KB) into a 3-stage ring that completes on an mbarrier; warps 0-7
// (4 row quarters x 2 column halves, 32 x 64 each) consume it with ldmatrix + mma.sync and hand the slot back through
// the `empty` barrier.  CTAs of one row tile are adjacent in launch order, so the X tile is read from HBM once and
// then served from L2.
constexpr int kBxBM = 128, kBxBN = 128, kBxBK = 64, kBxStages = 3, kBxThreads = 288;
constexpr int kBxBox = 128 * 128;   // one [128 rows][64 bf16] box

struct BxSmem {
    alignas(1024) unsigned char x[kBxStages][2][kBxBox];   // [stage][hi|lo]
    alignas(1024) unsigned char w[kBxStages][2][kBxBox];
    alignas(8) uint64_t full[kBxStages];
    uint64_t empty[kBxStages];
};

__global__ void __launch_bounds__(kBxThreads, 1)
k_gemm_bf16x3(const __grid_constant__ CUtensorMap tmXhi, const __grid_constant__ CUtensorMap tmXlo,
              const __grid_constant__ CUtensorMap tmWhi, const __grid_constant__ CUtensorMap tmWlo,
              const float *__restrict__ bias, float *__restrict__ Y, int64_t ldy, int M, int K, int nslices) {
    extern __shared__ __align__(1024) unsigned char tc_smem_raw[];
    BxSmem &sm = *reinterpret_cast<BxSmem *>(((uintptr_t)tc_smem_raw + 1023) & ~uintptr_t(1023));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = (int)(blockIdx.x % nslices) * kBxBN, m0 = (int)(blockIdx.x / nslices) * kBxBM;
    const int nkb = K / kBxBK;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kBxStages; s++) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();
    if (warp == 8) {
        // ===== TMA producer
        if (lane == 0) {
            tma_prefetch_desc(&tmXhi); tma_prefetch_desc(&tmXlo); tma_prefetch_desc(&tmWhi); tma_prefetch_desc(&tmWlo);
            for (int kb = 0; kb < nkb; kb++) {
                const int s = kb % kBxStages, n = kb / kBxStages;
                if (n > 0) mbar_wait(&sm.empty[s], (n - 1) & 1);
                mbar_expect_tx(&sm.full[s], 4 * kBxBox);
                tma_load_2d(sm.x[s][0], &tmXhi, kb * kBxBK, m0, &sm.full[s]);
                tma_load_2d(sm.x[s][1], &tmXlo, kb * kBxBK, m0, &sm.full[s]);
                tma_load_2d(sm.w[s][0], &tmWhi, kb * kBxBK, n0, &sm.full[s]);
                tma_load_2d(sm.w[s][1], &tmWlo, kb * kBxBK, n0, &sm.full[s]);
            }
        }
        return;
    }
    // ===== consumers: warp w owns rows [32 (w % 4), +32) and columns [64 (w / 4), +64) of the tile
    const int wm = (warp & 3) * 32, wn = (warp >> 2) * 64;
    float acc[2][8][4];
#pragma unroll
    for (int a = 0; a < 2; a++)
#pragma unroll
        for (int b = 0; b < 8; b++)
#pragma unroll
            for (int c = 0; c < 4; c++) acc[a][b][c] = 0.f;
    for (int kb = 0; kb < nkb; kb++) {
        const int s = kb % kBxStages;
        mbar_wait(&sm.full[s], (kb / kBxStages) & 1);
        warp_mma_sw128_k64<2>(smem_u32(sm.x[s][0]), smem_u32(sm.x[s][1]), smem_u32(sm.w[s][0]), smem_u32(sm.w[s][1]), wm, wn, acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);
    }
    // ===== epilogue: bias, fp32 pairs straight from the accumulator fragments (a lane quad covers 32 contiguous bytes)
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
        const int n = n0 + wn + 8 * nt + 2 * (lane & 3);
        const float2 bn = bias ? make_float2(__ldg(bias + n), __ldg(bias + n + 1)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int mt = 0; mt < 2; mt++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int m = m0 + wm + 16 * mt + (lane >> 2) + 8 * h;
                if (m < M)
                    *reinterpret_cast<float2 *>(Y + (int64_t)m * ldy + n) =
                        make_float2(acc[mt][nt][2 * h] + bn.x, acc[mt][nt][2 * h + 1] + bn.y);
            }
    }
}

// ------------------------------------------- fused depthwise -> 1x1 (tensor cores) -> ReLU ----
// Tensor-core version of k_dwpw (dfb_model.cu) at fp32-level accuracy (BF16x3): one CTA per 128-row tile.
//   0. thread 0 asks the TMA engine for every raw input (and pathway) frame of the tile -- one contiguous
//      Fin * 256-byte bulk copy per frame -- plus the pre-swizzled 16 KB weight image: the CTA's whole input is
//      in flight at once without passing through registers;
//   1. all 256 threads run the depthwise (+pathway) prologue out of shared memory (thread = channel quad x 8
//      consecutive rows), split the result x = hi + lo into BF16 planes and write them in the 128-byte swizzle
//      layout (a row of 64 channels is exactly one 128-byte row: conflict-free ldmatrix);
//   2. warp w multiplies rows [16 w, +16) by the 64 x 64 weight (ldmatrix + mma.sync; hi*hi + lo*hi + hi*lo), fp32
//      accumulators in registers;
//   3. bias, ReLU, and the fp32 tile is staged in the (now free) operand planes with an XOR chunk swizzle;
//   4. the CTA streams the staged tile out with coalesced 256-byte half-warp stores.
// Two CTAs per SM overlap each other's load / MMA / store phases.  Shared memory (1024-byte aligned base):
//   [0, 32K) A hi | lo planes (later the fp32 staging tile)   [32K, 48K) W hi | lo   [48K, 48K + raw) raw frames
//   then bias[64] and two mbarriers.
constexpr int kDxThreads = 256;
constexpr uint32_t kDxW = 32768, kDxRaw = 49152, kDxTail = 64 * 4 + 32;


// MASK = 1 (last ERB decoder block of the kt = 1 models): the tile holds whole frames, so the mask head
//   m[t,f] = sigmoid(sum_{df,c} w[df][c] * (relu(e0 * ps + pb) + out)[t][f+df-1][c] + bias)
// (conv0_out(conv0p(e0) + convt1(...)), deepfilternet3.py:253) is evaluated right on the staged fp32 tile and
// `out` itself never goes to HBM (p.out may be null).
template <int MODE, int KT, int PATH, int MASK>
__global__ void __launch_bounds__(kDxThreads, 2)
k_dwpw_bx(DwPwParams p, const float *__restrict__ w_sw /* [hi | lo] x [64 n][64 k] BF16, 128B-swizzled rows */) {
    extern __shared__ __align__(1024) unsigned char tc_smem_raw[];
    const uint32_t sb = smem_u32(tc_smem_raw);
    if (sb & 1023u) __trap();  // the swizzled operand planes need a 1024-byte aligned base
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.y, t0 = blockIdx.x * p.NF;
    const int nf = min(p.NF, p.T - t0);
    const int R = nf * p.Fout;  // rows actually present
    const int tq0 = t0 - (KT - 1);
    const uint32_t fbytes = (uint32_t)p.Fin * kCh * 4;
    const uint32_t raw_in = sb + kDxRaw, raw_path = raw_in + (uint32_t)(p.NF + KT - 1) * fbytes;
    const uint32_t raw_e0 = raw_in + (uint32_t)(p.NF + KT - 1) * fbytes * (PATH ? 2u : 1u);  // MASK: [NF][Fout][64]
    const uint32_t obytes = (uint32_t)p.Fout * kCh * 4;
    const uint32_t tail = raw_e0 + (MASK ? (uint32_t)p.NF * obytes : 0u);
    const uint32_t s_bias = tail, bar_raw = tail + 264;
    const uint32_t s_mask = raw_in;  // MASK: ps | pb | w[3][64], written over the raw input frames once they are converted
    if (tid == 0) {
        mbar_init_a(bar_raw, 1);
        fence_barrier_init();
        const int ta = max(tq0, 0), tb = t0 + nf;  // frames [ta, tb)
        mbar_expect_tx_a(bar_raw, (uint32_t)(tb - ta) * fbytes * (PATH ? 2u : 1u) + 2u * kCh * 128u + (MASK ? (uint32_t)nf * obytes : 0u));
        if (MASK)
            for (int t = t0; t < tb; t++)
                bulk_load(raw_e0 + (uint32_t)(t - t0) * obytes, p.mk_e0 + ((int64_t)b * p.T + t) * p.Fout * kCh, obytes, bar_raw);
        for (int t = ta; t < tb; t++) {
            bulk_load(raw_in + (uint32_t)(t - tq0) * fbytes, p.in + ((int64_t)b * p.T + t) * p.in_fs, fbytes, bar_raw);
            if (PATH) bulk_load(raw_path + (uint32_t)(t - tq0) * fbytes, p.path + ((int64_t)b * p.T + t) * p.path_fs, fbytes, bar_raw);
        }
        bulk_load(sb + kDxW, w_sw, 2 * kCh * 128, bar_raw);
    }
    if (tid < kCh / 4) sts128(s_bias + tid * 16, __ldg(reinterpret_cast<const float4 *>(p.bias) + tid));
    // ---- depthwise taps of this thread's channel quad, pathway affine
    const int cq = tid & 15, slot = tid >> 4;
    float4 wd[KT][3], ps4, pb4;
#pragma unroll
    for (int dt = 0; dt < KT; dt++)
#pragma unroll
        for (int df = 0; df < 3; df++) wd[dt][df] = __ldg(reinterpret_cast<const float4 *>(p.dw + (dt * 3 + df) * kCh) + cq);
    if (PATH) {
        ps4 = __ldg(reinterpret_cast<const float4 *>(p.ps) + cq);
        pb4 = __ldg(reinterpret_cast<const float4 *>(p.pb) + cq);
    }
    // rows r = 8 slot + i: (frame fr, bin fo) by multiply-shift division (exact for r < 128), then incrementally
    int fr = (8 * slot * p.fo_magic) >> 16, fo = 8 * slot - fr * p.Fout;
    __syncthreads();  // barriers initialised before anyone waits on them
    mbar_wait_a(bar_raw, 0);
    // ---- prologue
    auto rd = [&](uint32_t a) -> float4 {
        float4 x = lds128(a);
        if (PATH) {
            const float4 e = lds128(a + (raw_path - raw_in));
            x.x += fmaxf(fmaf(e.x, ps4.x, pb4.x), 0.f); x.y += fmaxf(fmaf(e.y, ps4.y, pb4.y), 0.f);
            x.z += fmaxf(fmaf(e.z, ps4.z, pb4.z), 0.f); x.w += fmaxf(fmaf(e.w, ps4.w, pb4.w), 0.f);
        }
        return x;
    };
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const int t_first = KT > 1 ? stream_first(p.first, b, p.w0) : 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int r = 8 * slot + i;
        float4 acc = zero4;
        if (r < R) {
#pragma unroll
            for (int dt = 0; dt < KT; dt++) {
                // tap dt reads frame t - (KT-1-dt) = raw frame fr + dt; before the start of the stream it is zero padding
                if (KT > 1 && tq0 + fr + dt < t_first) continue;
                const uint32_t fb = raw_in + (uint32_t)(fr + dt) * fbytes + cq * 16;
                if (MODE == DW_S1) {
                    const uint32_t a = fb + (uint32_t)fo * 256;
                    if (fo > 0) acc = f4_fma(rd(a - 256), wd[dt][0], acc);
                    acc = f4_fma(rd(a), wd[dt][1], acc);
                    if (fo + 1 < p.Fin) acc = f4_fma(rd(a + 256), wd[dt][2], acc);
                } else if (MODE == DW_S2) {
                    const uint32_t a = fb + (uint32_t)fo * 512;
                    if (fo > 0) acc = f4_fma(rd(a - 256), wd[dt][0], acc);
                    acc = f4_fma(rd(a), wd[dt][1], acc);
                    acc = f4_fma(rd(a + 256), wd[dt][2], acc);
                } else {  // DW_T2: out[2j] = w1 x[j]; out[2j+1] = w2 x[j] + w0 x[j+1]
                    const uint32_t a = fb + (uint32_t)(fo >> 1) * 256;
                    if ((fo & 1) == 0) {
                        acc = f4_fma(rd(a), wd[dt][1], acc);
                    } else {
                        acc = f4_fma(rd(a), wd[dt][2], acc);
                        if ((fo >> 1) + 1 < p.Fin) acc = f4_fma(rd(a + 256), wd[dt][0], acc);
                    }
                }
            }
        }
        uint32_t h0, l0, h1, l1;
        bf16x2_split(acc.x, acc.y, h0, l0);
        bf16x2_split(acc.z, acc.w, h1, l1);
        const uint32_t off = sb + sw128_off(r, cq >> 1) + (cq & 1) * 8;
        sts64(off, h0, h1);
        sts64(off + 16384, l0, l1);
        if (++fo == p.Fout) { fo = 0; fr++; }
    }
    __syncthreads();   // operand planes complete
    if (MASK && tid >= 64 && tid < 64 + 80) {  // ps | pb | w[3][64] as 80 float4
        const int i = tid - 64;
        const float4 *src = i < 16 ? reinterpret_cast<const float4 *>(p.mk_ps) + i
                          : i < 32 ? reinterpret_cast<const float4 *>(p.mk_pb) + (i - 16)
                                   : reinterpret_cast<const float4 *>(p.mk_w) + (i - 32);
        sts128(s_mask + i * 16, __ldg(src));
    }
    float acc[1][8][4];
#pragma unroll
    for (int nt = 0; nt < 8; nt++)
#pragma unroll
        for (int c = 0; c < 4; c++) acc[0][nt][c] = 0.f;
    warp_mma_sw128_k64<1>(sb, sb + 16384, sb + kDxW, sb + kDxW + 8192, warp * 16, 0, acc);
    __syncthreads();   // every warp has read its operand rows: the planes become the staging tile
    // ---- accumulator -> bias + ReLU -> staging tile (row r, 16-byte chunk j at r * 256 + ((j ^ (r & 15)) << 4))
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
        const int c = 8 * nt + 2 * (lane & 3);
        float b0, b1;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b0), "=f"(b1) : "r"(s_bias + 4 * c));
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int r = warp * 16 + (lane >> 2) + 8 * h;
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(sb + r * 256 + (((c >> 2) ^ (r & 15)) << 4) + (c & 3) * 4),
                         "f"(fmaxf(acc[0][nt][2 * h] + b0, 0.f)), "f"(fmaxf(acc[0][nt][2 * h + 1] + b1, 0.f)) : "memory");
        }
    }
    __syncthreads();
    if (MASK) {
        // thread = (channel quad j, 8 consecutive rows of one frame): X = relu(e0 * ps + pb) + out is formed once per
        // (row, quad), each row feeds the three taps of its neighbours, and the 16 quads are reduced with shuffles
        const int j = tid & 15, r0 = 8 * slot;
        const int fr = (r0 * p.fo_magic) >> 16, f0 = r0 - fr * p.Fout;   // Fout % 8 == 0: the 8 rows share a frame
        const float4 s4 = lds128(s_mask + j * 16), b4 = lds128(s_mask + 256 + j * 16);
        const float4 w0 = lds128(s_mask + 512 + j * 16), w1 = lds128(s_mask + 512 + 256 + j * 16), w2 = lds128(s_mask + 512 + 512 + j * 16);
        float part[8];
#pragma unroll
        for (int i = 0; i < 8; i++) part[i] = 0.f;
        if (r0 < R) {
#pragma unroll
            for (int i = -1; i <= 8; i++) {
                const int f2 = f0 + i, r2 = r0 + i;
                if (f2 < 0 || f2 >= p.Fout) continue;
                const float4 d = lds128(sb + r2 * 256 + ((j ^ (r2 & 15)) << 4));
                const float4 e = lds128(raw_e0 + r2 * 256 + j * 16);
                float4 x;
                x.x = fmaxf(fmaf(e.x, s4.x, b4.x), 0.f) + d.x; x.y = fmaxf(fmaf(e.y, s4.y, b4.y), 0.f) + d.y;
                x.z = fmaxf(fmaf(e.z, s4.z, b4.z), 0.f) + d.z; x.w = fmaxf(fmaf(e.w, s4.w, b4.w), 0.f) + d.w;
                // row r2 is tap df = 0 of output r2 + 1, tap 1 of r2, tap 2 of r2 - 1
                if (i + 1 < 8) part[i + 1 < 0 ? 0 : i + 1] += x.x * w0.x + x.y * w0.y + x.z * w0.z + x.w * w0.w;
                if (i >= 0 && i < 8) part[i < 0 ? 0 : (i > 7 ? 7 : i)] += x.x * w1.x + x.y * w1.y + x.z * w1.z + x.w * w1.w;
                if (i - 1 >= 0) part[i - 1 > 7 ? 7 : i - 1] += x.x * w2.x + x.y * w2.y + x.z * w2.z + x.w * w2.w;
            }
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            float v = part[i];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            part[i] = v;
        }
        if (r0 < R && j < 8) {
            float z = part[0];
#pragma unroll
            for (int i = 1; i < 8; i++) z = j == i ? part[i] : z;
            z += __ldg(p.mk_bias);
            p.mk_out[((int64_t)b * p.T + t0 + fr) * p.Fout + f0 + j] = 1.f / (1.f + expf(-z));
        }
    }
    // ---- coalesced write-out: half a warp per 256-byte row, 8 consecutive rows per thread
    if (p.out || p.out_hi) {
        const int j = tid & 15;
        int fr2 = (8 * slot * p.fo_magic) >> 16, fo2 = 8 * slot - fr2 * p.Fout;
        int64_t off = ((int64_t)b * p.T + t0 + fr2) * p.out_fs + fo2 * kCh + j * 4;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int r = 8 * slot + i;
            if (r < R) {
                const float4 v = lds128(sb + r * 256 + ((j ^ (r & 15)) << 4));
                if (p.out) *reinterpret_cast<float4 *>(p.out + off) = v;
                if (p.out_hi) {
                    uint32_t h0, l0, h1, l1;
                    bf16x2_split(v.x, v.y, h0, l0);
                    bf16x2_split(v.z, v.w, h1, l1);
                    *reinterpret_cast<uint2 *>(p.out_hi + off) = make_uint2(h0, h1);
                    *reinterpret_cast<uint2 *>(p.out_lo + off) = make_uint2(l0, l1);
                }
            }
            off += kCh;
            if (++fo2 == p.Fout) { fo2 = 0; off += p.out_fs - (int64_t)p.Fout * kCh; }
        }
    }
}

template <int MODE, int KT, int PATH, int MASK = 0>
static int launch_dwpw_bx(cudaStream_t s, const DwPwParams &p, const float *w_sw, int B) {
    static int attr_smem[64] = {0};  // per device: largest dynamic shared memory size set so far
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    const int raw = (p.NF + KT - 1) * p.Fin * kCh * 4 * (PATH ? 2 : 1) + (MASK ? p.NF * p.Fout * kCh * 4 : 0);
    const int smem = (int)kDxRaw + raw + (int)kDxTail;
    if (smem > 227 * 1024) return fail(DFB_ERR_UNSUPPORTED, "dwpw tile needs %d bytes of shared memory", smem);
    if (smem > attr_smem[dev]) {
        DFB_CUDA(cudaFuncSetAttribute(k_dwpw_bx<MODE, KT, PATH, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_smem[dev] = smem;
    }
    dim3 grid((unsigned)((p.T + p.NF - 1) / p.NF), (unsigned)B);
    DFB_PROF("k_dwpw_bx", s);
    k_dwpw_bx<MODE, KT, PATH, MASK><<<grid, kDxThreads, smem, s>>>(p, w_sw);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

template <int MODE>
int launch_dwpw_tc(cudaStream_t s, DwPwParams p, const float *w_sw, int B) {
    p.NF = 128 / p.Fout;
    if (p.NF < 1) p.NF = 1;
    if (p.NF * p.Fout > 128) return fail(DFB_ERR_UNSUPPORTED, "dwpw tile: Fout = %d", p.Fout);
    p.fo_magic = (65536 + p.Fout - 1) / p.Fout;
    for (int r = 0; r < 128; r++)
        if (((r * p.fo_magic) >> 16) != r / p.Fout) return fail(DFB_ERR_UNSUPPORTED, "dwpw tile: Fout = %d", p.Fout);
    if ((p.in_fs * 4) % 16 || (p.path && (p.path_fs * 4) % 16)) return fail(DFB_ERR_UNSUPPORTED, "dwpw: unaligned frame stride");
    const bool path = p.path != nullptr;
    if (MODE == DW_S1) {
        if (p.kt == 1) return path ? launch_dwpw_bx<DW_S1, 1, 1>(s, p, w_sw, B) : launch_dwpw_bx<DW_S1, 1, 0>(s, p, w_sw, B);
        if (p.kt == 2) return path ? launch_dwpw_bx<DW_S1, 2, 1>(s, p, w_sw, B) : launch_dwpw_bx<DW_S1, 2, 0>(s, p, w_sw, B);
    } else if (MODE == DW_S2 && !path) {
        if (p.kt == 1) return launch_dwpw_bx<DW_S2, 1, 0>(s, p, w_sw, B);
        if (p.kt == 2) return launch_dwpw_bx<DW_S2, 2, 0>(s, p, w_sw, B);
    } else if (MODE == DW_T2 && path && p.kt == 1) {
        if (p.mk_e0) {
            return launch_dwpw_bx<DW_T2, 1, 1, 1>(s, p, w_sw, B);
        }
        return launch_dwpw_bx<DW_T2, 1, 1>(s, p, w_sw, B);
    }
    return fail(DFB_ERR_UNSUPPORTED, "dwpw tensor-core path: mode %d kt %d path %d", MODE, p.kt, (int)path);
}
template int launch_dwpw_tc<DW_S1>(cudaStream_t, DwPwParams, const float *, int);
template int launch_dwpw_tc<DW_S2>(cudaStream_t, DwPwParams, const float *, int);
template int launch_dwpw_tc<DW_T2>(cudaStream_t, DwPwParams, const float *, int);

// ---------------------------------------------------------- DF pathway conv on tensor cores ----
// coefs[b,t,f,:] = relu( pw( conv_t(c0) ) + b )  (df_convp, deepfilternet3.py:293-295: grouped (2) temporal conv 64 -> 10
// with kernel (KTP,1), 1x1 conv 10 x 10, BN, ReLU; KTP = 5 for DeepFilterNet2 / 3, 3 for DeepFilterNet2_ll, and
// instances for every KTP from 1 to 5).  On FFMA this conv is instruction-issue bound (~250 warp instructions
// per frame and bin pair at KTP = 5), so the channel contraction runs on the tensor pipe:
//   Y[t, g*32 + dt*5 + o] = sum_{c in group g} w1[dt][g*5+o][c] * c0[t, f, c]        (one [128 t x 64 c] x [64 c x 64] product)
//   z[t, g*5 + o]         = sum_dt Y[t - (KTP - 1) + dt, g*32 + dt*5 + o]             (shifted adds out of shared memory)
//   coefs[t, f, :]        = relu(z . w2 + b)
// One CTA = (stream, bin f, 124 output frames): its 128 time rows of c0[., f, :] (KTP - 1 <= 4 frames of history; every
// KTP keeps the 124-frame tile, so the launch geometry does not depend on it) arrive as two TMA
// tensor boxes (rows 24.5 KB apart in HBM, 2 x 128 B per row, 128-byte swizzle), are split into BF16 hi / lo operand planes
// (BF16x3: fp32-level accuracy), each warp multiplies 16 of the rows by the 64 x 64 weight with mma.sync and stages its part
// of Y in shared memory (row stride 51 floats) and 128 threads (one per time row) do the shifted sums, the 1x1 conv and the 40-byte store.
constexpr int kCvThreads = 256, kCvOut = 124, kCvYld = 51 /* 2 x 25 used columns + 1 */, kCvBins = 8;
// shared memory: [0, 32K) A hi | lo planes, [32K, 48K) W hi | lo, [48K, 80K) raw fp32 boxes of the current bin,
// [80K, +26112) the staged Y tile, then w2 | bias and the barriers
constexpr uint32_t kCvW = 32768, kCvRawOff = 49152, kCvYs = kCvRawOff + 32768, kCvTail = kCvYs + 128 * kCvYld * 4;

struct CvParams {
    const float *w_sw;   // [hi | lo] x [64 n][64 k] BF16, 128B-swizzled rows: n = g*32 + dt*5 + o, k = channel
    const float *w2;     // [10 in][10 out]
    const float *bias;   // [10]
    float *coefs;        // [B,T,Fd,10]
    int T, Fd;
    const int64_t *first;   // streaming slots: first frame of each stream (stream_first), or null
    int64_t w0;
};

// One CTA = (stream, kCvBins consecutive bins, 124 output frames): the weight image and the barrier set-up are paid once
// per CTA, and the TMA load of the next bin's rows is issued as soon as the current bin's rows have
// been converted, so it overlaps the MMA and the epilogue (the first version ran one bin per CTA: 0.39 of HBM).
template <int ORDER, int KTP>
__global__ void __launch_bounds__(kCvThreads, 2) k_df_convp_tc(const __grid_constant__ CUtensorMap tmC0, CvParams p) {
    constexpr int O2 = 2 * ORDER, NY = KTP * ORDER;
    extern __shared__ __align__(1024) unsigned char tc_smem_raw[];
    const uint32_t sb = (smem_u32(tc_smem_raw) + 1023u) & ~1023u;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int f_begin = blockIdx.x * kCvBins, f_end = min(f_begin + kCvBins, p.Fd);
    const int b = blockIdx.z, t0 = blockIdx.y * kCvOut, r0 = t0 - (KTP - 1);
    const uint32_t s_w2 = sb + kCvTail, bar_raw = s_w2 + 512, bar_w = bar_raw + 16;
    const int row = b * p.T + r0;   // may be negative for the first stream: out-of-bounds rows arrive as zeros
    auto load_bin = [&](int f) {    // thread 0 only
        mbar_expect_tx_a(bar_raw, 32768);
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                     ::"r"(sb + kCvRawOff), "l"((uint64_t)&tmC0), "r"(f * 64), "r"(row), "r"(bar_raw) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                     ::"r"(sb + kCvRawOff + 16384), "l"((uint64_t)&tmC0), "r"(f * 64 + 32), "r"(row), "r"(bar_raw) : "memory");
    };
    if (tid == 0) {
        mbar_init_a(bar_raw, 1);
        mbar_init_a(bar_w, 1);
        fence_barrier_init();
        mbar_expect_tx_a(bar_w, 16384);
        bulk_load(sb + kCvW, p.w_sw, 16384, bar_w);
        load_bin(f_begin);
    }
    for (int i = tid; i < O2 * O2 + O2; i += kCvThreads)
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(s_w2 + 4 * i), "f"(i < O2 * O2 ? __ldg(p.w2 + i) : __ldg(p.bias + i - O2 * O2)) : "memory");
    __syncthreads();
    mbar_wait_a(bar_w, 0);
    const int r = tid & 127, half = tid >> 7;
    // before the start of the stream (for b > 0 the box holds the previous stream's rows; a slot's stream may start inside
    // the window)
    const bool zero = r0 + r < stream_first(p.first, b, p.w0);
    for (int f = f_begin, it = 0; f < f_end; f++, it++) {
        const uint32_t par = (uint32_t)(it & 1);
        mbar_wait_a(bar_raw, par);
        {   // fp32 rows -> BF16 hi / lo operand planes: thread = (time row, channel half)
            const uint32_t src = sb + kCvRawOff + (uint32_t)half * 16384u + (uint32_t)r * 128u;
            // all eight loads first: the shared-memory accesses are volatile asm statements, so a load placed after a store
            // in program order also waits for it -- as one loop every chunk paid the load latency (short-scoreboard was the
            // top stall of this kernel)
            float4 xs[8];
#pragma unroll
            for (int c = 0; c < 8; c++) xs[c] = lds128(src + (uint32_t)((c ^ (r & 7)) << 4));
#pragma unroll
            for (int c = 0; c < 8; c++) {
                float4 x = xs[c];
                if (zero) x = make_float4(0.f, 0.f, 0.f, 0.f);
                uint32_t h0, l0, h1, l1;
                bf16x2_split(x.x, x.y, h0, l0);
                bf16x2_split(x.z, x.w, h1, l1);
                const int cq = half * 8 + c;
                const uint32_t off = sb + sw128_off(r, cq >> 1) + (cq & 1) * 8;
                sts64(off, h0, h1);
                sts64(off + 16384, l0, l1);
            }
        }
        fence_proxy_async();  // the raw boxes were read through the generic proxy before the TMA engine refills them
        __syncthreads();     // planes complete (and the raw boxes free; the previous bin's epilogue has left the Y tile)
        if (tid == 0 && f + 1 < f_end) load_bin(f + 1);   // overlaps the MMA and the epilogue below
        {   // Y rows [16 warp, +16) -> shared memory; column n = g * 32 + j of the product is Y[., g * NY + j] for j < NY
            float acc[1][8][4];
#pragma unroll
            for (int nt = 0; nt < 8; nt++)
#pragma unroll
                for (int c = 0; c < 4; c++) acc[0][nt][c] = 0.f;
            warp_mma_sw128_k64<1>(sb, sb + 16384, sb + kCvW, sb + kCvW + 8192, warp * 16, 0, acc);
#pragma unroll
            for (int nt = 0; nt < 8; nt++)
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int n = 8 * nt + 2 * (lane & 3) + (e & 1), g = n >> 5, j = n & 31;
                    const int rr = warp * 16 + (lane >> 2) + 8 * (e >> 1);
                    if (j < NY)
                        asm volatile("st.shared.f32 [%0], %1;" ::"r"(sb + kCvYs + (uint32_t)(rr * kCvYld + g * NY + j) * 4u), "f"(acc[0][nt][e]) : "memory");
                }
        }
        __syncthreads();     // Y staged
        if (tid < 128) {
            const int t = r0 + tid;
            if (tid >= KTP - 1 && tid < KTP - 1 + kCvOut && t < p.T) {
                float z[O2];
#pragma unroll
                for (int g = 0; g < 2; g++)
#pragma unroll
                    for (int o = 0; o < ORDER; o++) {
                        float a = 0.f;
#pragma unroll
                        for (int dt = 0; dt < KTP; dt++) {
                            float y;
                            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(y) : "r"(sb + kCvYs + (uint32_t)((tid - (KTP - 1) + dt) * kCvYld + g * NY + dt * ORDER + o) * 4u));
                            a += y;
                        }
                        z[g * ORDER + o] = a;
                    }
                float outv[O2];
#pragma unroll
                for (int qo = 0; qo < O2; qo++) {
                    float a;
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(a) : "r"(s_w2 + 4 * (O2 * O2 + qo)));
#pragma unroll
                    for (int k = 0; k < O2; k++) {
                        float w;
                        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(w) : "r"(s_w2 + 4 * (k * O2 + qo)));
                        a = fmaf(z[k], w, a);
                    }
                    outv[qo] = fmaxf(a, 0.f);
                }
                float *dst = p.coefs + (((int64_t)b * p.T + t) * p.Fd + f) * O2;   // 40-byte rows: 8-byte aligned
#pragma unroll
                for (int qo = 0; qo < O2; qo += 2) *reinterpret_cast<float2 *>(dst + qo) = make_float2(outv[qo], outv[qo + 1]);
            }
        }
        // the next iteration's conversion writes the operand planes (read by the MMAs that completed above) and its
        // __syncthreads orders this bin's shifted sums before the next Y tile is staged
    }
}

// ================================================================ tensor-core GRU recurrence ====
// torch.nn.GRU cell (DeepFilterNet/df/modules.py:684,723), hidden size HH = 256 or 512.  A cluster of HH / 32 CTAs owns
// NS streams for the whole sequence; CTA `rank` owns 32 hidden units, i.e. the 96 W_hh rows (3 gates x 32 units) of
// them, kept on chip for the whole kernel as a BF16 hi / lo split (W = hi + lo to ~2^-17): the hi plane in registers
// (the mma.sync A fragments), the lo plane in shared memory (ldmatrix, XOR-swizzled rows).  Per time step the
// 6 x (HH / 128) MMA warps -- 16 rows x 128 k each -- multiply the hidden state of the group (the B operand in shared
// memory: [NS streams][HH], BF16 hi / lo, core matrices of 8 x 16 B ordered so that a CTA's 32 units are one
// contiguous piece) with mma.sync (hi*hi + lo*hi + hi*lo, fp32 accumulate) and leave their K-partial sums in shared
// memory; one thread per (unit pair, stream) adds them up, applies the gates in fp32, writes the CTA's slice of the new
// state and broadcasts it to the peers -- one bulk DSMEM copy per peer (cp.async.bulk shared::cta -> shared::cluster)
// or, XG = 1, one TMA multicast of a global scratch piece -- that completes bytes on each receiver's mbarrier, so no
// cluster barrier or fence sits on the step's critical path.  The fp32 hidden state of a thread's own units stays in
// registers; only the MMA operand is BF16.
namespace cg = cooperative_groups;

constexpr int kGtU = 32, kGtRows = 3 * kGtU;   // hidden units / W_hh rows per CTA (both hidden sizes)
// h operand (B, K-major) as 8 x 16 B core matrices ordered [k core matrix][row group][hi|lo][8 rows x 16 B]: a CTA's 32
// units (4 k core matrices) are one contiguous piece (2 KB for 16 streams) -> one bulk copy per peer.
// NS = streams per cluster (MMA N): 16 (lowest step latency), 32 or 48 (fewer clusters for large batches; H = 256 only --
// at H = 512 the state buffers of 32 streams and the W_hh lo plane do not fit next to each other in shared memory).
template <int NS, int HH>
struct GtCfg {
    static constexpr int kC = HH / kGtU;              // CTAs per cluster: 8 / 16
    static constexpr int kKS = HH / 128;              // K quarters of 128 per W_hh row: 2 / 4
    static constexpr int kMmaWarps = 6 * kKS;         // 16-row tile x K slice of 128
    static constexpr int kGateThreads = 16 * NS;      // one per (unit pair, stream)
    static constexpr int kThreads = kGateThreads > 32 * kMmaWarps ? kGateThreads : 32 * kMmaWarps;
    static constexpr int kLbo = (NS / 8) * 256;       // stride between K-adjacent core matrices
    static constexpr int kSbo = 256;                  // stride between 8-stream row groups
    static constexpr int kPlane = 128;                // hi -> lo
    static constexpr int kPiece = 4 * kLbo;           // one CTA's slice
    static constexpr int kBuf = (HH / 8) * kLbo;      // one buffer
    static constexpr int kPreLd = NS + 1;             // row stride of the partial sums
};

template <int NS, int HH>
struct GruTcSmem {
    alignas(1024) unsigned char h[2][GtCfg<NS, HH>::kBuf];   // [buffer][k core matrix][row group][hi|lo][8 rows x 16 B]
    alignas(128) unsigned char wlo[kGtRows * HH * 2];         // W_hh lo plane [96 rows][HH], 16-byte chunk j of row r at j ^ (r & 7)
    float pre[GtCfg<NS, HH>::kKS][kGtRows][GtCfg<NS, HH>::kPreLd];   // K-partial sums of W_hh h
    alignas(8) uint64_t bar_h[2];
};

struct GruTcParams {
    const float *xproj;  // [B,T,3H]
    const float *whh;    // [3H][H]
    const float *bhh;    // [3H]
    const float *res;    // optional [B,T,H], added to the OUTPUT only
    float *hout;         // [B,T,H], or null: only the planes are wanted
    unsigned short *hout_hi, *hout_lo;  // optional BF16 hi/lo planes of hout (A operand of the next projection GEMM)
    int planes_res;      // 1: the planes hold hout + res (input of a grouped linear), 0: the residual-free h
    // time-chunked execution: steps t = 0 .. T-1 are frames t0 + t of buffers holding Ts frames per stream; the
    // recurrence starts from h0 [B][H] (null: zeros) and leaves its final state in hT [B][H] (may alias h0)
    const float *h0;
    float *hT;
    int t0, Ts;
    int B, T, Bc;
    long long *dbg;      // optional [T][8] clock64 stamps of CTA 0, thread 0 (0 step start, 1 state arrived, 2 MMAs done,
                         // 3 gates done, 4 slice sent)
    unsigned char *xbuf; // (XG) exchange scratch in global memory [cluster][2][CTA][kPiece]
    // streaming slots: first frame of each stream (stream_first; step t is window frame t0 + t), or null.  The state holds
    // h = 0 through the steps before it: those frames do not exist for the stream.
    const int64_t *first;
    int64_t w0;
    // (HOLD) run flags [B][Ts]: step t of stream b runs when run[b * Ts + t0 + t] != 0; a held step keeps the state as it
    // was, exchanges it and writes it out as that step's output
    const unsigned char *run;
};

// XG = 1: the new state travels through L2 instead of SM to SM -- every CTA stores its slice to a global scratch piece and
// asks the TMA engine for ONE multicast bulk copy of that piece into all CTAs of the cluster (itself included) instead of
// kC - 1 per-peer DSMEM copies.
template <int NS, int HH, int XG, int HOLD>
__global__ void __launch_bounds__(GtCfg<NS, HH>::kThreads, 1) k_gru_tc(GruTcParams p) {
    using Cfg = GtCfg<NS, HH>;
    constexpr int kGtThreads = Cfg::kThreads, kGtH = HH, kGtC = Cfg::kC, NT = NS / 8;
    extern __shared__ __align__(1024) unsigned char tc_smem_raw[];
    GruTcSmem<NS, HH> &sm = *reinterpret_cast<GruTcSmem<NS, HH> *>(((uintptr_t)tc_smem_raw + 1023) & ~uintptr_t(1023));
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank();
    const int group = blockIdx.x / kGtC;
    const int b0 = group * p.Bc;
    const int nb = min(p.Bc, p.B - b0);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int H = kGtH, T = p.T;
    for (int i = tid; i < (int)sizeof(sm.h) / 16; i += kGtThreads) reinterpret_cast<uint4 *>(&sm.h[0][0])[i] = make_uint4(0, 0, 0, 0);  // h0 = 0
    if (tid == 0) {
        mbar_init(&sm.bar_h[0], XG ? 1 : 2);   // thread 0's expect_tx arrive (+ one gate-warp arrive: own slice written)
        mbar_init(&sm.bar_h[1], XG ? 1 : 2);
        fence_barrier_init();
    }
    if (p.h0) {  // carried state: every CTA builds the whole operand h_{-1} of its streams in buffer 0
        __syncthreads();   // after the zero fill
        for (int i = tid; i < nb * (kGtH / 2); i += kGtThreads) {
            const int s = i / (kGtH / 2), gu = (i - s * (kGtH / 2)) * 2;
            const float2 hv = *reinterpret_cast<const float2 *>(p.h0 + (int64_t)(b0 + s) * kGtH + gu);
            unsigned short h0b, l0b, h1b, l1b;
            bf16_split(hv.x, h0b, l0b);
            bf16_split(hv.y, h1b, l1b);
            const uint32_t off = (uint32_t)((gu >> 3) * Cfg::kLbo + (s >> 3) * Cfg::kSbo + (s & 7) * 16 + (gu & 7) * 2);
            *reinterpret_cast<uint32_t *>(sm.h[0] + off) = h0b | (uint32_t)h1b << 16;
            *reinterpret_cast<uint32_t *>(sm.h[0] + off + Cfg::kPlane) = l0b | (uint32_t)l1b << 16;
        }
    }
    // ---- W_hh slice: MMA warp (mt, kq) = rows [16 mt, +16) (row rho = gate * 32 + unit), k [128 kq, +128).  Its A
    //      fragments of the hi plane stay in registers; the lo plane goes to shared memory.
    const bool mma_warp = warp < Cfg::kMmaWarps;
    const int mt = warp % 6, kq = warp / 6;
    uint32_t wa[8][4];
    const uint32_t wlo = smem_u32(sm.wlo);
    if (mma_warp) {
#pragma unroll
        for (int ks = 0; ks < 8; ks++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
                // fragment register e: row g + 8 (e & 1), k pair 2 q + 8 (e >> 1) of the 16 x 16 tile
                const int rho = 16 * mt + (lane >> 2) + 8 * (e & 1), k = 128 * kq + 16 * ks + 2 * (lane & 3) + 8 * (e >> 1);
                const int gate = rho / kGtU, u = rho - gate * kGtU;
                const float2 w = *reinterpret_cast<const float2 *>(p.whh + ((int64_t)gate * H + rank * kGtU + u) * H + k);
                uint32_t hi, lo;
                bf16x2_split(w.x, w.y, hi, lo);
                wa[ks][e] = hi;
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(wlo + (uint32_t)rho * (HH * 2) + ((((k >> 3) ^ (rho & 7))) << 4) + (k & 7) * 2),
                             "r"(lo) : "memory");
            }
    }
    fence_proxy_async();   // the zeroed / carried state buffers are overwritten by bulk copies later
    __syncthreads();
    cluster.sync();  // every CTA's barriers are initialised and its h buffers zeroed before any remote copy
    const uint32_t step_bytes = (uint32_t)((kGtC - (XG ? 0 : 1)) * Cfg::kPiece);  // one piece from each of the peers (XG: and the own one)

    // gate thread: unit pair up = tid % 16 (units 2 up, 2 up + 1 of this CTA), stream s = tid / 16
    const int up = tid & 15, s = tid >> 4;
    const bool gate_thread = tid < Cfg::kGateThreads;
    const bool active = gate_thread && s < nb;
    const int gu = rank * kGtU + 2 * up;       // first of the two global hidden units of this thread
    float hprev0 = 0.f, hprev1 = 0.f;
    float2 bhr = make_float2(0.f, 0.f), bhz = bhr, bhn = bhr;
    int t_first = 0;   // first step of this stream (steps before it keep h = 0)
    if (active) {
        t_first = stream_first(p.first, b0 + s, p.w0) - p.t0;
        if (p.h0) {
            const float2 hv = *reinterpret_cast<const float2 *>(p.h0 + (int64_t)(b0 + s) * H + gu);
            hprev0 = hv.x; hprev1 = hv.y;
        }
        bhr = *reinterpret_cast<const float2 *>(p.bhh + gu);
        bhz = *reinterpret_cast<const float2 *>(p.bhh + H + gu);
        bhn = *reinterpret_cast<const float2 *>(p.bhh + 2 * H + gu);
    }
    // byte offset of this (stream, unit pair) inside an h buffer (hi plane): core matrix gu / 8, row group s / 8
    const uint32_t hoff = (uint32_t)((gu >> 3) * Cfg::kLbo + (s >> 3) * Cfg::kSbo + (s & 7) * 16 + (gu & 7) * 2);
    const uint32_t piece0 = (uint32_t)(rank * Cfg::kPiece);  // this CTA's slice of a buffer
    const bool dbg_on = p.dbg && blockIdx.x == 0 && tid == 0;
    const int mat = lane >> 3, rr = lane & 7;
    for (int t = 0; t < T; t++) {
        const int cur = t & 1;
        if (dbg_on) p.dbg[t * 8 + 0] = clock64();
        if (tid == 0 && t + 1 < T) mbar_expect_tx(&sm.bar_h[cur ^ 1], step_bytes);
        float2 xr = make_float2(0.f, 0.f), xz = xr, xn = xr;
        bool held = false;
        if (active) {
            if (HOLD) held = p.run[(int64_t)(b0 + s) * p.Ts + p.t0 + t] == 0;
            const float *xp = p.xproj + ((int64_t)(b0 + s) * p.Ts + p.t0 + t) * (3 * H) + gu;
            xr = *reinterpret_cast<const float2 *>(xp);
            xz = *reinterpret_cast<const float2 *>(xp + H);
            xn = *reinterpret_cast<const float2 *>(xp + 2 * H);
            // xproj streams from HBM (3 KB per frame and stream, used once): pull the rows of frame t + 3 into L2 now, so
            // that the loads above are L2 hits by the time they are issued
            if (t + 3 < T && (up & 7) == 0) {   // two requests per 128-byte line (16 threads x 8 bytes cover a gate's 32 units)
                const float *xq = xp + 3 * (3 * H);
                asm volatile("prefetch.global.L2 [%0];" ::"l"(xq));
                asm volatile("prefetch.global.L2 [%0];" ::"l"(xq + H));
                asm volatile("prefetch.global.L2 [%0];" ::"l"(xq + 2 * H));
            }
        }
        if (t > 0) mbar_wait(&sm.bar_h[cur], (uint32_t)(((t - 1) >> 1) & 1));
        if (dbg_on) p.dbg[t * 8 + 1] = clock64();
        if (mma_warp) {
            // ===== partial pre-activations W_hh[16 mt .., 128 kq ..] . h[cur] -> sm.pre[kq]
            float acc[NT][4];
#pragma unroll
            for (int n = 0; n < NT; n++) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
            const uint32_t hb = smem_u32(sm.h[cur]);
#pragma unroll
            for (int ks = 0; ks < 8; ks++) {
                const int k = 128 * kq + 16 * ks;
                uint32_t al[4];
                {   // matrices: rows 0-7 | 8-15, k 0-7 | 8-15
                    const int r = 16 * mt + rr + ((mat & 1) << 3);
                    ldsm_x4(wlo + (uint32_t)r * (HH * 2) + ((((k >> 3) + (mat >> 1)) ^ (r & 7)) << 4), al);
                }
#pragma unroll
                for (int n = 0; n < NT; n++) {
                    // matrices: k core matrix k / 8 | k / 8 + 1 of row group n, hi plane | lo plane
                    uint32_t b[4];
                    ldsm_x4(hb + (uint32_t)(((k >> 3) + (mat & 1)) * Cfg::kLbo + n * Cfg::kSbo + (mat >> 1) * Cfg::kPlane + rr * 16), b);
                    mma_bf16x3(acc[n], wa[ks], al, b[0], b[1], b[2], b[3]);
                }
            }
#pragma unroll
            for (int n = 0; n < NT; n++)
#pragma unroll
                for (int e = 0; e < 4; e++)
                    sm.pre[kq][16 * mt + (lane >> 2) + 8 * (e >> 1)][8 * n + 2 * (lane & 3) + (e & 1)] = acc[n][e];
        }
        __syncthreads();   // partial sums complete (and every MMA warp is done with h[cur])
        if (dbg_on) p.dbg[t * 8 + 2] = clock64();
        uint32_t vhi = 0, vlo = 0;
        if (active) {
            const int u0 = 2 * up;
            float a[6];
#pragma unroll
            for (int g = 0; g < 3; g++) {
                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int q = 0; q < Cfg::kKS; q++) { s0 += sm.pre[q][g * kGtU + u0][s]; s1 += sm.pre[q][g * kGtU + u0 + 1][s]; }
                a[2 * g] = s0; a[2 * g + 1] = s1;
            }
            const float r0 = gt_sigmoid(xr.x + a[0] + bhr.x), r1 = gt_sigmoid(xr.y + a[1] + bhr.y);
            const float z0 = gt_sigmoid(xz.x + a[2] + bhz.x), z1 = gt_sigmoid(xz.y + a[3] + bhz.y);
            const float n0 = gt_tanh(xn.x + r0 * (a[4] + bhn.x)), n1 = gt_tanh(xn.y + r1 * (a[5] + bhn.y));
            const float k0 = hprev0, k1 = hprev1;
            hprev0 = (1.f - z0) * n0 + z0 * hprev0;
            hprev1 = (1.f - z1) * n1 + z1 * hprev1;
            if (t < t_first) hprev0 = hprev1 = 0.f;
            if (HOLD && held) { hprev0 = k0; hprev1 = k1; }
            unsigned short h0, l0, h1, l1;
            bf16_split(hprev0, h0, l0);
            bf16_split(hprev1, h1, l1);
            vhi = h0 | (uint32_t)h1 << 16;
            vlo = l0 | (uint32_t)l1 << 16;
            if (t + 1 < T) {
                if (XG) {   // own piece of the scratch buffer (same layout as the shared-memory slice)
                    unsigned char *xp = p.xbuf + ((size_t)(group * 2 + (cur ^ 1)) * kGtC + rank) * Cfg::kPiece + (hoff - piece0);
                    *reinterpret_cast<uint32_t *>(xp) = vhi;
                    *reinterpret_cast<uint32_t *>(xp + Cfg::kPlane) = vlo;
                } else {
                    *reinterpret_cast<uint32_t *>(sm.h[cur ^ 1] + hoff) = vhi;
                    *reinterpret_cast<uint32_t *>(sm.h[cur ^ 1] + hoff + Cfg::kPlane) = vlo;
                }
            }
        }
        if (dbg_on) p.dbg[t * 8 + 3] = clock64();
        // own slice (generic stores) -> visible to the bulk-copy proxy
        if (t + 1 < T) { if (XG) fence_proxy_async_global(); else fence_proxy_async(); }
        __syncthreads();   // slice written, partial sums read (the next step's MMAs may overwrite them)
        if (t + 1 < T) {
            if (XG) {
                if (tid == 0) {
                    const unsigned char *xp = p.xbuf + ((size_t)(group * 2 + (cur ^ 1)) * kGtC + rank) * Cfg::kPiece;
                    bulk_load_multicast(smem_u32(sm.h[cur ^ 1]) + piece0, xp, Cfg::kPiece, smem_u32(&sm.bar_h[cur ^ 1]),
                                        (uint16_t)((1u << kGtC) - 1u));
                }
            } else if (lane == 0) {
                // warp w copies the CTA's slice to peers w, w + #warps, ... (skipping itself); warp 0 also signals the local
                // barrier
                const uint32_t src = smem_u32(sm.h[cur ^ 1]) + piece0;
                for (int j = warp; j < kGtC - 1; j += kGtThreads / 32) {
                    const int peer = j + (j >= rank ? 1 : 0);
                    dsmem_bulk_copy(mapa_u32(src, peer), src, Cfg::kPiece, mapa_u32(smem_u32(&sm.bar_h[cur ^ 1]), peer));
                }
                if (warp == 0) mbar_arrive(&sm.bar_h[cur ^ 1]);  // own slice is in place
            }
        }
        if (dbg_on) p.dbg[t * 8 + 4] = clock64();
        if (active) {  // global result last: nothing on the recurrence's critical path waits for it
            const int64_t o = ((int64_t)(b0 + s) * p.Ts + p.t0 + t) * H + gu;
            float2 ov = make_float2(hprev0, hprev1);
            if (p.hT && t + 1 == T) *reinterpret_cast<float2 *>(p.hT + (int64_t)(b0 + s) * H + gu) = ov;
            if (p.res) { const float2 rv = *reinterpret_cast<const float2 *>(p.res + o); ov.x += rv.x; ov.y += rv.y; }
            if (p.hout) *reinterpret_cast<float2 *>(p.hout + o) = ov;
            if (p.hout_hi) {  // residual-free h (the next layer's projection input) or the layer output
                if (p.planes_res && p.res) bf16x2_split(ov.x, ov.y, vhi, vlo);
                *reinterpret_cast<uint32_t *>(p.hout_hi + o) = vhi;
                *reinterpret_cast<uint32_t *>(p.hout_lo + o) = vlo;
            }
        }
    }
    cluster.sync();  // no CTA exits while peers may still address its shared memory
}

// exchange scratch of the XG variant: one buffer per (device, stream) -- launches on one stream are serialised, the two
// decoders' recurrences run on different streams
static unsigned char *gru_xbuf(cudaStream_t s, size_t bytes) {
    struct Ent { unsigned char *p = nullptr; size_t cap = 0; };
    static std::mutex mu;
    static std::map<std::pair<int, cudaStream_t>, Ent> pool;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    Ent &e = pool[{dev, s}];
    if (e.cap < bytes) {
        if (e.p) { cudaDeviceSynchronize(); cudaFree(e.p); e.p = nullptr; e.cap = 0; }
        const size_t want = (bytes + (1u << 20)) & ~size_t((1u << 20) - 1);
        if (cudaMalloc(&e.p, want) != cudaSuccess) { e.p = nullptr; return nullptr; }
        e.cap = want;
    }
    return e.p;
}

// function attributes (once per device) and the launch configuration of one k_gru_tc instance; `at` backs cfg.attrs
template <int NS, int HH, int XG, int HOLD = 0>
static int gru_tc_config(cudaLaunchConfig_t &cfg, cudaLaunchAttribute (&at)[1]) {
    using Cfg = GtCfg<NS, HH>;
    static PerDeviceOnce attr_once;
    const int smem = (int)sizeof(GruTcSmem<NS, HH>) + 1024;
    if (auto once_guard = attr_once.first()) {
        if (Cfg::kC > 8) DFB_CUDA(cudaFuncSetAttribute(k_gru_tc<NS, HH, XG, HOLD>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        DFB_CUDA(cudaFuncSetAttribute(k_gru_tc<NS, HH, XG, HOLD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    }
    cfg = cudaLaunchConfig_t{};
    cfg.blockDim = dim3(Cfg::kThreads);
    cfg.dynamicSmemBytes = smem;
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = Cfg::kC; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return DFB_OK;
}

// clusters of one k_gru_tc instance that can be resident at once on the current device (cached per device)
template <int NS, int HH, int XG>
static int gru_tc_max_clusters(int *out) {
    static std::atomic<int> cached[64];
    int dev = 0;
    DFB_CUDA(cudaGetDevice(&dev));
    int n = cached[dev & 63].load(std::memory_order_relaxed);
    if (n <= 0) {
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute at[1];
        int rc = gru_tc_config<NS, HH, XG>(cfg, at);
        if (rc) return rc;
        cfg.gridDim = dim3((unsigned)GtCfg<NS, HH>::kC);
        DFB_CUDA(cudaOccupancyMaxActiveClusters(&n, k_gru_tc<NS, HH, XG, 0>, &cfg));
        cached[dev & 63].store(n, std::memory_order_relaxed);
    }
    *out = n;
    return DFB_OK;
}

template <int NS, int HH, int XG>
static int launch_gru_tc_n(cudaStream_t s, GruTcParams p) {
    using Cfg = GtCfg<NS, HH>;
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at[1];
    int rc = p.run ? gru_tc_config<NS, HH, XG, 1>(cfg, at) : gru_tc_config<NS, HH, XG, 0>(cfg, at);
    if (rc) return rc;
    p.Bc = NS;
    const int ngroups = (p.B + NS - 1) / NS;
    cfg.gridDim = dim3((unsigned)(ngroups * Cfg::kC));
    cfg.stream = s;
    if (XG) {
        p.xbuf = gru_xbuf(s, (size_t)ngroups * 2 * Cfg::kC * Cfg::kPiece);
        if (!p.xbuf) return fail(DFB_ERR_OOM, "GRU exchange scratch");
    }
    DFB_PROF(HH == 256 ? "k_gru_tc" : "k_gru_tc512", s);
    if (p.run) DFB_CUDA(cudaLaunchKernelEx(&cfg, k_gru_tc<NS, HH, XG, 1>, p));
    else DFB_CUDA(cudaLaunchKernelEx(&cfg, k_gru_tc<NS, HH, XG, 0>, p));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return DFB_OK;
}

// The instance (streams per cluster, exchange) the recurrence runs for B streams of hidden size H.  wide != 0: 32 streams
// per cluster when the batch needs more than 4 clusters of 16 (see GtCfg).  H = 512: clusters of 16 CTAs with 16 streams.
static int gru_tc_select(int B, int H, int wide, int *ns, int *xg_out) {
    static const int force = getenv("DFB_GRU_NS") ? atoi(getenv("DFB_GRU_NS")) : 0;
    // exchange through L2 + multicast (k_gru_tc XG): bit 0: H = 512, bit 1: H = 256 / 32 streams, bit 2: H = 256 / 16 streams.
    // Default: all.
    static const int xg = getenv("DFB_GRU_XG") ? atoi(getenv("DFB_GRU_XG")) : 7;
    if (H == 512) { *ns = 16; *xg_out = xg & 1; return DFB_OK; }
    if (H != 256) return fail(DFB_ERR_UNSUPPORTED, "tensor-core recurrence: hidden size %d", H);
    // 16 streams per cluster have the shortest step but more cluster time per stream: once a launch needs several waves of
    // the co-resident clusters anyway, 32 per cluster are faster
    const bool use32 = force ? force == 32 : ((wide && B > 64) || B >= 256);
    // beyond one wave of 32-stream clusters (as many as the device can hold at once), 48 streams per cluster (N = 48, 768
    // threads) need fewer clusters, so that 512 streams stay in one wave
    static const int no48 = getenv("DFB_GRU_NO48") ? atoi(getenv("DFB_GRU_NO48")) : 0;
    if (use32 && !force && !no48) {
        int wave = 0, rc = gru_tc_max_clusters<32, 256, 1>(&wave);
        if (rc) return rc;
        if (B > wave * 32) { *ns = 48; *xg_out = 1; return DFB_OK; }
    }
    *ns = use32 ? 32 : 16;
    *xg_out = (xg & (use32 ? 2 : 4)) ? 1 : 0;
    return DFB_OK;
}

// ns = 0, xg = -1: the instance gru_tc_select picks; otherwise instance <ns, H, xg>, DFB_ERR_UNSUPPORTED when it is not built
int launch_gru_tc(cudaStream_t s, const float *xproj, const float *whh, const float *bhh, const float *res, float *hout,
                  unsigned short *hout_hi, unsigned short *hout_lo, int B, int T, long long *dbg, int wide, int planes_res,
                  const GruWindow *w, int H, int ns, int xg) {
    if (!hout && !hout_hi) return fail(DFB_ERR_INVALID, "tensor-core recurrence: neither an fp32 output nor planes");
    GruTcParams p{xproj, whh, bhh, res, hout, hout_hi, hout_lo, planes_res, w ? w->h0 : nullptr, w ? w->hT : nullptr,
                  w ? w->t0 : 0, w ? w->Ts : T, B, T, 0, dbg};
    p.first = w ? w->first : nullptr;
    p.w0 = w ? w->w0 : 0;
    p.run = w ? w->run : nullptr;
    if (ns == 0 && xg == -1) {
        const int rc = gru_tc_select(B, H, wide, &ns, &xg);
        if (rc) return rc;
    }
    if (xg == 0 || xg == 1) {
        if (H == 512 && ns == 16) return xg ? launch_gru_tc_n<16, 512, 1>(s, p) : launch_gru_tc_n<16, 512, 0>(s, p);
        if (H == 256 && ns == 16) return xg ? launch_gru_tc_n<16, 256, 1>(s, p) : launch_gru_tc_n<16, 256, 0>(s, p);
        if (H == 256 && ns == 32) return xg ? launch_gru_tc_n<32, 256, 1>(s, p) : launch_gru_tc_n<32, 256, 0>(s, p);
        if (H == 256 && ns == 48 && xg) return launch_gru_tc_n<48, 256, 1>(s, p);
    }
    return fail(DFB_ERR_UNSUPPORTED, "tensor-core recurrence: instance NS %d H %d XG %d is not built", ns, H, xg);
}

int cached_map_f32_sw128(CUtensorMap *out, const void *base, int64_t rows, int64_t cols, int64_t ld, int box_rows);

bool df_convp_built(int order, int kt) { return order == 5 && kt >= 1 && kt <= 5; }

template <int ORDER, int KTP>
static int launch_df_convp_kt(cudaStream_t s, const CUtensorMap &mc, const CvParams &p, int B) {
    const int smem = 1024 + (int)kCvTail + 512 + 64;
    static PerDeviceOnce attr_once;
    if (auto once_guard = attr_once.first())
        DFB_CUDA(cudaFuncSetAttribute(k_df_convp_tc<ORDER, KTP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    // every KTP keeps the 124-frame output tile: the 128 staged rows hold at least KTP - 1 <= 4 rows of history
    dim3 grid((unsigned)((p.Fd + kCvBins - 1) / kCvBins), (unsigned)((p.T + kCvOut - 1) / kCvOut), (unsigned)B);
    DFB_PROF("k_df_convp_tc", s);
    k_df_convp_tc<ORDER, KTP><<<grid, kCvThreads, smem, s>>>(mc, p);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

// c0 [B,T,Fd,64] -> coefs [B,T,Fd,10] (pathway term), tensor-core version; w_sw: host-packed operand image (weights.py)
int launch_df_convp_tc(cudaStream_t s, const float *c0, const float *w_sw, const float *w2, const float *bias, float *coefs, int B, int T,
                       int Fd, int order, int kt, const int64_t *first, int64_t w0) {
    if (!df_convp_built(order, kt))
        return fail(DFB_ERR_UNSUPPORTED, "df_order %d / df_pathway_kernel_size_t %d (built kernels: df_order 5, kt 1-5)", order, kt);
    if ((int64_t)B * T >= (int64_t(1) << 31) - 256 || B > 65535) return fail(DFB_ERR_UNSUPPORTED, "df pathway conv: batch too large for one launch");
    CUtensorMap mc;
    int rc;
    if ((rc = cached_map_f32_sw128(&mc, c0, (int64_t)B * T, (int64_t)Fd * kCh, (int64_t)Fd * kCh, 128))) return rc;
    const CvParams p{w_sw, w2, bias, coefs, T, Fd, first, w0};
    switch (kt) {
        case 1: return launch_df_convp_kt<5, 1>(s, mc, p, B);
        case 2: return launch_df_convp_kt<5, 2>(s, mc, p, B);
        case 3: return launch_df_convp_kt<5, 3>(s, mc, p, B);
        case 4: return launch_df_convp_kt<5, 4>(s, mc, p, B);
        default: return launch_df_convp_kt<5, 5>(s, mc, p, B);
    }
}

// ------------------------------------------------------------------------------- host side ----
int cached_map_bf16(CUtensorMap *out, const void *base, int64_t rows, int64_t cols, int64_t ld, int box_rows);  // dfb_gl.cu

// Y[M,N] = X . W^T + bias with X, W given as BF16 hi/lo planes (X: [M][K] pitch ldx, W: [N][K] pitch K)
int launch_gemm_bf16x3(cudaStream_t s, const void *x_hi, const void *x_lo, int64_t ldx, const void *w_hi, const void *w_lo,
                       const float *bias, float *y, int64_t ldy, int64_t M, int N, int K) {
    if (N % kBxBN || K % kBxBK || (ldx % 8) || M <= 0 || ldy % 2 || ((uintptr_t)w_hi & 15) || ((uintptr_t)w_lo & 15))
        return fail(DFB_ERR_UNSUPPORTED, "bf16x3 GEMM shape M=%lld N=%d K=%d", (long long)M, N, K);
    const int nslices = N / kBxBN;
    const int64_t ntiles = (M + kBxBM - 1) / kBxBM;
    if (ntiles * nslices > 0x7fffffff) return fail(DFB_ERR_UNSUPPORTED, "bf16x3 GEMM: M = %lld", (long long)M);
    CUtensorMap mxh, mxl, mwh, mwl;
    int rc;
    // (cached per (base, shape): the arenas hand out the same addresses call after call)
    if ((rc = cached_map_bf16(&mxh, x_hi, M, K, ldx, kBxBM)) || (rc = cached_map_bf16(&mxl, x_lo, M, K, ldx, kBxBM)) ||
        (rc = cached_map_bf16(&mwh, w_hi, N, K, K, kBxBN)) || (rc = cached_map_bf16(&mwl, w_lo, N, K, K, kBxBN)))
        return rc;
    static PerDeviceOnce attr_once;
    const int smem = (int)sizeof(BxSmem) + 1024;
    if (auto once_guard = attr_once.first()) DFB_CUDA(cudaFuncSetAttribute(k_gemm_bf16x3, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DFB_PROF("k_gemm_bf16x3[gru_proj]", s);
    k_gemm_bf16x3<<<(unsigned)(ntiles * nslices), kBxThreads, smem, s>>>(mxh, mxl, mwh, mwl, bias, y, ldy, (int)M, K, nslices);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

}  // namespace dfb

// Debug aid (tests/test_gpu_gru_tc.py): one k_gru_tc launch on caller-given device pointers
extern "C" int dfb_debug_gru_tc(const float *xproj, const float *whh, const float *bhh, const float *res, float *hout,
                                void *hout_hi, void *hout_lo, int planes_res, const float *h0, float *hT, const int64_t *first,
                                int64_t w0, int t0, int Ts, int B, int T, int H, int ns, int xg, void *stream) {
    if (!xproj || !whh || !bhh || (!hout && !hout_hi) || (!hout_hi != !hout_lo))
        return dfb::fail(DFB_ERR_INVALID, "gru_tc: null argument");
    if (B <= 0 || T <= 0 || t0 < 0 || (int64_t)t0 + T > Ts)
        return dfb::fail(DFB_ERR_INVALID, "gru_tc: B %d, window [%d, %d + %d) of %d frames", B, t0, t0, T, Ts);
    const dfb::GruWindow w{h0, hT, t0, Ts, first, w0};
    return dfb::launch_gru_tc((cudaStream_t)stream, xproj, whh, bhh, res, hout, (unsigned short *)hout_hi,
                              (unsigned short *)hout_lo, B, T, nullptr, 0, planes_res, &w, H, ns, xg);
}

// Debug aid (tests/test_gpu_gating_runtime.py): dfb_debug_gru_tc with run flags run [B][Ts] (k_gru_tc's HOLD instances)
extern "C" int dfb_debug_gru_tc_hold(const float *xproj, const float *whh, const float *bhh, const float *res, float *hout,
                                     void *hout_hi, void *hout_lo, int planes_res, const float *h0, float *hT, const int64_t *first,
                                     int64_t w0, const unsigned char *run, int t0, int Ts, int B, int T, int H, int ns, int xg,
                                     void *stream) {
    if (!xproj || !whh || !bhh || !run || (!hout && !hout_hi) || (!hout_hi != !hout_lo))
        return dfb::fail(DFB_ERR_INVALID, "gru_tc_hold: null argument");
    if (B <= 0 || T <= 0 || t0 < 0 || (int64_t)t0 + T > Ts)
        return dfb::fail(DFB_ERR_INVALID, "gru_tc_hold: B %d, window [%d, %d + %d) of %d frames", B, t0, t0, T, Ts);
    const dfb::GruWindow w{h0, hT, t0, Ts, first, w0, run};
    return dfb::launch_gru_tc((cudaStream_t)stream, xproj, whh, bhh, res, hout, (unsigned short *)hout_hi,
                              (unsigned short *)hout_lo, B, T, nullptr, 0, planes_res, &w, H, ns, xg);
}

// Debug aid (tests/test_gpu_gru_tc.py): one k_gemm_bf16x3 launch on caller-given device pointers
extern "C" int dfb_debug_gemm_bf16x3(const void *x_hi, const void *x_lo, int64_t ldx, const void *w_hi, const void *w_lo,
                                     const float *bias, float *y, int64_t ldy, int64_t M, int N, int K, void *stream) {
    if (!x_hi || !x_lo || !w_hi || !w_lo || !y) return dfb::fail(DFB_ERR_INVALID, "gemm_bf16x3: null argument");
    return dfb::launch_gemm_bf16x3((cudaStream_t)stream, x_hi, x_lo, ldx, w_hi, w_lo, bias, y, ldy, M, N, K);
}

// Debug aid (tests/test_gpu_dfn2_ll.py): one k_df_convp_tc launch on caller-given device pointers
extern "C" int dfb_debug_df_convp_tc(const float *c0, const float *w_sw, const float *w2, const float *bias, float *coefs, int B,
                                     int T, int Fd, int order, int kt, const int64_t *first, int64_t w0, void *stream) {
    if (!c0 || !w_sw || !w2 || !bias || !coefs) return dfb::fail(DFB_ERR_INVALID, "df_convp_tc: null argument");
    if (B <= 0 || T <= 0 || Fd <= 0) return dfb::fail(DFB_ERR_INVALID, "df_convp_tc: B %d, T %d, Fd %d", B, T, Fd);
    return dfb::launch_df_convp_tc((cudaStream_t)stream, c0, w_sw, w2, bias, coefs, B, T, Fd, order, kt, first, w0);
}
