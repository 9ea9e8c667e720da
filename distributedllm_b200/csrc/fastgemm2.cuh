// fastgemm2.cuh -- K2: the prefill weight matmul on the Hopper tensor cores ("fast mode"), a wgmma tile kernel fed by TMA.
//
//   Y[token][row] = sum_k  W[row][k] * X[token][k]      W: Q4_0 or Q8_0 (packed layout of kernels.cuh), X: fp16 activations
//
//   * CTA tile 128 weight rows x 256 tokens (two consumer warpgroups, each 64 rows x 256 tokens as two wgmma m64n128k16
//     accumulators, 128 fp32 registers a thread), or 128 tokens for narrow matrices (twice the CTAs);
//   * the producer lane streams the raw quantised weights of one 128-row quad with a 1-D TMA bulk copy -- the same
//     bytes per block of HBM traffic as the decode kernel, nothing is dequantised in HBM -- and the activation tile
//     through the tensor-map TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B: the hardware writes the K-major layout the GMMA
//     descriptor expects);
//   * 8 dequant warps expand the weights to fp16 IN SHARED MEMORY in that layout (Q4_0 nibbles and Q8_0 int8 through the
//     fp16 magic-number conversion, one HMUL2 by the block scale); each warpgroup dequantises its own 64 rows, issues
//     their wgmma and keeps one K block in flight while it dequantises the next;
//   * the fused epilogue (store | +residual | SiLU-gate) runs straight from the accumulator registers.
// Numerics ("fast mode", tolerance-checked, NOT bit-exact): activations go through the reference's Q8_0 quantisation
// (k_prep_q8_f16) and both operands are rounded to fp16 (<= 2^-11 relative each); products are exact in fp32 and
// accumulated in fp32 in hardware order.  Measured: 2.7e-4 relative RMS on one matmul; ~5e-3 per layer on hidden states,
// dominated by Q8_0 codes of the NEXT matmul's input flipping by one step (tests/test_gpu_fast_prefill.py).
// Reference for the operation: ggml_compute_forward_mul_mat (ggml.c:10577-10749); the CUDA analogue in the reference tree
// is dequantise -> cublasSgemm (ggml-cuda.cu:2514-2560).
#pragma once
#include <cuda.h>

#include "kernels.cuh"

namespace b200 {

// ---- activation pre-pass: [RMSNorm * w ->] Q8_0 quantise -> dequantise -> fp16 row (one warp per 32-block) --------
struct PrepArgs { const float * x; int ldx; const float * norm_w; uint16_t * xh; int K, N; };

template <bool NORM>
__global__ void __launch_bounds__(256) k_prep_q8_f16(const PrepArgs a) {
    __shared__ double red[8];
    grid_dep_wait();
    const int n = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float * x = a.x + (size_t) n * a.ldx;
    float scale = 1.f;
    if (NORM) {
        // fast mode is checked against a tolerance, not bit for bit: the tree sum's scale is used as it is (exact mode
        // certifies it, see rms_scale)
        double s = 0.0;
        for (int i = tid; i < a.K; i += 256) s += (double) fmul(x[i], x[i]);
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[warp] = s;
        __syncthreads();
        double tot = 0.0;
        for (int i = 0; i < 8; i++) tot += red[i];
        scale = __fdiv_rn(1.0f, __fsqrt_rn(fadd((float)(tot / (double) a.K), 1e-6f)));
    }
    for (int b = warp; b < a.K / 32; b += 8) {
        float v = x[b * 32 + lane];
        if (NORM) v = fmul(fmul(v, scale), a.norm_w[b * 32 + lane]);
        float amax = fabsf(v);
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float d = h2f(f2h(__fdiv_rn(amax, 127.f)));
        const float id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
        const float q = (float) rint_small(fmul(v, id));
        a.xh[(size_t) n * a.K + b * 32 + lane] = f2h(fmul(q, d));
    }
}

// ---- wgmma helpers -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) {
    // K-major, SWIZZLE_128B, 8-row groups 1024 B apart (sm_90 GMMA descriptor: start>>4 | LBO 1 | SBO 64 | layout 1 = 128B swizzle)
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t) 1 << 16) | ((uint64_t) 64 << 32) | ((uint64_t) 1 << 62);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence()  { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across an in-flight wgmma
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
    #pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i]) :: "memory");
}
// D[64 x 128] += A[64 x 16] * B[128 x 16]^T: fp16 operands K-major in shared memory, fp32 accumulator in the registers of
// the issuing warpgroup (thread t holds rows 16*(t/32) + (t%32)/4 + {0, 8}, columns 8*j + 2*(t%4) + {0, 1} as d[4j + 2i + c])
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1, 0, 0; }"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "n"(1)
                 : "memory");
}

enum { FG_STORE = 0, FG_RESID = 1, FG_GATE = 2 };

// Epilogue of one 64 x 128 accumulator block (layout of wgmma_m64n128k16): this thread holds rows m0 and m0 + 8 of the
// 128-row M tile (packed order) for the token pairs tok0 + 8j + {0, 1}.
template <int EPI, class Args>
__device__ __forceinline__ void gmma_epilogue(const Args & a, const float (&d)[64], int mt, int m0, int tok0) {
    #pragma unroll
    for (int j = 0; j < 16; j++) {
        #pragma unroll
        for (int c = 0; c < 2; c++) {
            const int tok = tok0 + 8 * j + c;
            if (tok >= a.N) continue;
            if (EPI == FG_GATE) {
                // packed G=2 order: row-groups alternate w1 / w3, so row m0 (w1, bit 3 clear) pairs with row m0 + 8 (w3)
                const int row = (mt * 8 + (m0 >> 4)) * 8 + (m0 & 7);
                if (row < a.out_rows) a.y[(size_t) tok * a.ldy + row] = fmul(h2f(a.tsilu[f2h(d[4 * j + c])]), d[4 * j + 2 + c]);
            } else {
                #pragma unroll
                for (int i = 0; i < 2; i++) {
                    const int row = mt * 128 + m0 + 8 * i;
                    float val = d[4 * j + 2 * i + c];
                    if (row < a.out_rows) {
                        if (EPI == FG_RESID) val = fadd(val, a.resid[(size_t) tok * a.ldr + row]);
                        a.y[(size_t) tok * a.ldy + row] = val;
                    }
                }
            }
        }
    }
}

constexpr int kF2M = 128, kF2K = 128;                      // token-tile width NT = 256 (wide matrices) or 128 (narrow ones: twice the CTAs)
constexpr int kF2DqWarps = 8;
constexpr int kF2Threads = (kF2DqWarps + 1) * 32;          // + TMA warp
constexpr int kF2ABytes = kF2M * kF2K * 2;                  // 32 KB: two [128 x 64] K-major SW128 sub-tiles
__host__ __device__ constexpr int f2_raw_bytes(int wt) { return 16 * chunk_bytes(wt); }                   // one quad of 128 rows
__host__ __device__ constexpr int f2_stage_bytes(int wt, int nt) { return ((f2_raw_bytes(wt) + 1023) & ~1023) + kF2ABytes + nt * kF2K * 2; }
__host__ __device__ constexpr int f2_stages(int wt, int nt) { return (nt == 128 && wt == kWT_Q4_0) ? 3 : 2; }
__host__ __device__ constexpr int f2_smem(int wt, int nt) { return f2_stages(wt, nt) * f2_stage_bytes(wt, nt) + 128; }   // Q8_0, NT 256: 231 552 of 232 448 B

struct FastGemm2Args {
    PackedW W;
    const float * resid; int ldr;
    float * y; int ldy;
    int N, out_rows;
    const uint16_t * tsilu;
};

__device__ __forceinline__ void tma_load_2d(void * dst, const CUtensorMap * map, int c0, int c1, uint64_t * bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

template <int WT, int EPI, int NT>
__global__ void __launch_bounds__(kF2Threads, 1) k_gemm_tc2(const FastGemm2Args a, const __grid_constant__ CUtensorMap xmap) {
    constexpr int CB = (WT == kWT_Q4_0) ? kQ4Chunk : kQ8Chunk;
    constexpr int kF2N = NT, kF2BBytes = NT * kF2K * 2, kF2Stages = f2_stages(WT, NT);
    constexpr int RAW = 16 * CB, RAWP = (RAW + 1023) & ~1023, STAGE = RAWP + kF2ABytes + kF2BBytes;
    extern __shared__ __align__(1024) uint8_t smem[];       // SWIZZLE_128B tiles need 1 KB alignment (no static shared memory in this kernel)
    uint64_t * bars = (uint64_t *)(smem + kF2Stages * STAGE);
    uint64_t * tma_full = bars, * stage_free = bars + 3;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int mt = blockIdx.x, nt = blockIdx.y;             // 128-row tile, 256-token tile
    const int nbq = a.W.nbq;
    const int TRp = a.W.TR;                                 // row-groups per packed tile (4 or 8)
    const int tiles_per_m = 16 / TRp;                       // packed tiles per 128 rows (16 row-groups)

    if (tid == 0) {
        // a stage is free once both consumer warpgroups have retired the wgmma group that read it
        for (int s = 0; s < kF2Stages; s++) { mbar_init(&tma_full[s], 1); mbar_init(&stage_free[s], 2); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == kF2DqWarps) {
        // -------------------------------------------------------------------- TMA producer (one thread)
        if (lane == 0) {
            grid_dep_launch();
            grid_dep_wait();                                 // the activation tile is the previous kernel's output
            const uint32_t per_tile = (uint32_t) TRp * CB;
            for (int kb = 0; kb < nbq; kb++) {
                const int s = kb % kF2Stages, use = kb / kF2Stages;
                if (use > 0) mbar_wait(&stage_free[s], (use - 1) & 1);
                uint8_t * stage = smem + (size_t) s * STAGE;
                mbar_arrive_expect_tx(&tma_full[s], (uint32_t)(RAW + kF2BBytes));
                for (int t = 0; t < tiles_per_m; t++) {
                    const uint8_t * src = a.W.data + (long long)(mt * tiles_per_m + t) * a.W.tile_bytes + (size_t) kb * per_tile;
                    bulk_g2s(stage + (size_t) t * per_tile, src, per_tile, &tma_full[s]);
                }
                // activations: tokens nt*256 .. +255, K block kb -> two [256 rows x 64 halfs] boxes, written SWIZZLE_128B
                uint8_t * B = stage + RAWP + kF2ABytes;
                tma_load_2d(B, &xmap, kb * kF2K, nt * kF2N, &tma_full[s]);
                tma_load_2d(B + kF2N * 128, &xmap, kb * kF2K + 64, nt * kF2N, &tma_full[s]);
            }
        }
    } else {
        // -------------------------------------------------------------------- two dequant + MMA warpgroups (256 threads)
        const int wg = warp >> 2;                            // warpgroup wg dequantises and multiplies rows 64*wg .. +63
        float acc[NT / 128][64];
        #pragma unroll
        for (int n = 0; n < NT / 128; n++)
            #pragma unroll
            for (int i = 0; i < 64; i++) acc[n][i] = 0.f;
        const int r8 = lane >> 2, w = lane & 3;
        for (int kb = 0; kb < nbq; kb++) {
            const int s = kb % kF2Stages, use = kb / kF2Stages;
            uint8_t * stage = smem + (size_t) s * STAGE;
            uint8_t * A = stage + RAWP;
            mbar_wait(&tma_full[s], use & 1);
            // this warp expands row-groups 2*warp, 2*warp+1 (rows 16*warp .. +15) of the quad
            #pragma unroll
            for (int gi = 0; gi < 2; gi++) {
                const int g = warp * 2 + gi;                 // row-group 0..15 of the M tile, in packed order
                const uint8_t * ch = stage + (size_t) g * CB;
                const uint4 wv = *(const uint4 *)(ch + lane * 16);
                uint4 wv2 = make_uint4(0, 0, 0, 0); uint2 sc;
                if (WT == kWT_Q8_0) { wv2 = *(const uint4 *)(ch + 512 + lane * 16); sc = *(const uint2 *)(ch + 1024 + r8 * 8); }
                else sc = *(const uint2 *)(ch + 512 + r8 * 8);
                const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
                const uint32_t ww2[4] = {wv2.x, wv2.y, wv2.z, wv2.w};
                const uint32_t sw[2] = {sc.x, sc.y};
                const int row = g * 8 + r8;                  // row within the 128-row tile (packed order)
                #pragma unroll
                for (int bq = 0; bq < 4; bq++) {
                    const uint32_t dh = (sw[bq >> 1] >> (16 * (bq & 1))) & 0xFFFFu;
                    const __half2 d2 = __halves2half2(__ushort_as_half((unsigned short) dh), __ushort_as_half((unsigned short) dh));
                    uint32_t lo0, lo1, hi0, hi1;             // e0 e1 | e2 e3 (k = 4w ..) and e16 e17 | e18 e19
                    if (WT == kWT_Q4_0) {
                        const uint32_t x = ww[bq] ^ 0x88888888u;             // back to offset-binary nibbles n = v + 8
                        const __half2 off = __halves2half2(__ushort_as_half((unsigned short) 0x6408), __ushort_as_half((unsigned short) 0x6408));   // 1032.0
                        uint32_t h[4];                        // {e0,e2} {e16,e18} {e1,e3} {e17,e19} relative to 4w
                        #pragma unroll
                        for (int i = 0; i < 4; i++) {
                            const uint32_t m = ((x >> (4 * i)) & 0x000F000Fu) | 0x64006400u;      // 1024 + n, exact in fp16
                            const __half2 v = __hmul2(__hsub2(*(const __half2 *) &m, off), d2);     // (n - 8) * d, one rounding
                            h[i] = *(const uint32_t *) &v;
                        }
                        lo0 = __byte_perm(h[0], h[2], 0x5410); lo1 = __byte_perm(h[0], h[2], 0x7632);
                        hi0 = __byte_perm(h[1], h[3], 0x5410); hi1 = __byte_perm(h[1], h[3], 0x7632);
                    } else {
                        // int8 q -> offset-binary u = q + 128 -> fp16 1024 + u (exact) -> minus 1152 -> times d
                        const __half2 off = __halves2half2(__ushort_as_half((unsigned short) 0x6480), __ushort_as_half((unsigned short) 0x6480));   // 1152.0
                        const uint32_t ul = ww[bq] ^ 0x80808080u, uh = ww2[bq] ^ 0x80808080u;
                        const uint32_t m0 = __byte_perm(ul, 0x64646464u, 0x4140), m1 = __byte_perm(ul, 0x64646464u, 0x4342);
                        const uint32_t m2 = __byte_perm(uh, 0x64646464u, 0x4140), m3 = __byte_perm(uh, 0x64646464u, 0x4342);
                        const __half2 v0 = __hmul2(__hsub2(*(const __half2 *) &m0, off), d2), v1 = __hmul2(__hsub2(*(const __half2 *) &m1, off), d2);
                        const __half2 v2 = __hmul2(__hsub2(*(const __half2 *) &m2, off), d2), v3 = __hmul2(__hsub2(*(const __half2 *) &m3, off), d2);
                        lo0 = *(const uint32_t *) &v0; lo1 = *(const uint32_t *) &v1; hi0 = *(const uint32_t *) &v2; hi1 = *(const uint32_t *) &v3;
                    }
                    const int klo = bq * 32 + 4 * w, khi = klo + 16;                      // k within the 128-wide block
                    {
                        const int sub = klo >> 6, kk = klo & 63, c8 = kk >> 3, within = (kk & 7) * 2;
                        *(uint2 *)(A + sub * (kF2M * 128) + row * 128 + ((c8 ^ (row & 7)) << 4) + within) = make_uint2(lo0, lo1);
                    }
                    {
                        const int sub = khi >> 6, kk = khi & 63, c8 = kk >> 3, within = (kk & 7) * 2;
                        *(uint2 *)(A + sub * (kF2M * 128) + row * 128 + ((c8 ^ (row & 7)) << 4) + within) = make_uint2(hi0, hi1);
                    }
                }
            }
            fence_proxy_async();                             // generic-proxy writes -> visible to the tensor core's async proxy
            named_bar_sync(1 + wg, 128);                     // this warpgroup's 64 rows of A are complete
            // A stage is rewritten only after the wgmma group that last read it (K block kb - stages) was retired below
            const uint32_t a_addr = smem_u32(A) + wg * (64 * 128), b_addr = smem_u32(stage + RAWP + kF2ABytes);
            wgmma_fence();
            #pragma unroll
            for (int n = 0; n < NT / 128; n++) acc_fence(acc[n]);
            #pragma unroll
            for (int k16 = 0; k16 < 8; k16++) {
                const uint32_t off = (k16 & 3) * 32;                                         // 32 B per K step of 16 inside the 128 B swizzle atom
                #pragma unroll
                for (int n = 0; n < NT / 128; n++)
                    wgmma_m64n128k16(acc[n], gmma_desc_k_sw128(a_addr + (k16 >> 2) * (kF2M * 128) + off),
                                     gmma_desc_k_sw128(b_addr + (k16 >> 2) * (kF2N * 128) + n * (128 * 128) + off));
            }
            wgmma_commit();
            wgmma_wait<1>();                                 // K block kb-1 retired: its stage may be refilled
            #pragma unroll
            for (int n = 0; n < NT / 128; n++) acc_fence(acc[n]);
            if (kb > 0 && (tid & 127) == 0) mbar_arrive(&stage_free[(kb - 1) % kF2Stages]);
        }
        wgmma_wait<0>();
        #pragma unroll
        for (int n = 0; n < NT / 128; n++) acc_fence(acc[n]);
        // -------------------------------------------------------------------- epilogue: registers -> global
        #pragma unroll
        for (int n = 0; n < NT / 128; n++)
            gmma_epilogue<EPI>(a, acc[n], mt, wg * 64 + (warp & 3) * 16 + r8, nt * kF2N + n * 128 + 2 * w);
    }
}

}  // namespace b200
