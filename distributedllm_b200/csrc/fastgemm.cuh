// fastgemm.cuh -- K2: prefill weight matmul on the Hopper tensor cores ("fast mode").
//
//   Y[token][row] = sum_k  W[row][k] * X[token][k]        W: Q4_0 (packed layout of kernels.cuh), X: activations
//
// wgmma.mma_async (m64n128k16, f16 x f16 -> f32) with the fp32 accumulator in the registers of one warpgroup:
//   * the producer lane streams the packed Q4_0 chunks of four 32-row tiles (= one 128-row M tile) with 1-D TMA bulk
//     copies into a raw ring -- the same 18 B/block HBM traffic as the decode kernel, nothing is dequantised in HBM;
//   * the four warps of the consumer warpgroup expand each 4-block quad to fp16 IN SHARED MEMORY, writing the K-major
//     SWIZZLE_128B layout the GMMA shared-memory descriptor expects (fp16 magic-number nibble conversion, one HMUL2 by
//     the block scale), and copy the matching activation tile; `fence.proxy.async` hands the tiles to the async proxy;
//   * the same warpgroup then issues 2 x 8 wgmma per 128-wide K block (rows 0..63 and 64..127, 128 accumulator registers
//     a thread) and keeps one K block in flight while it dequantises the next; after the last K block it applies the
//     fused epilogue straight from the accumulator registers (store | +residual | SiLU-gate).
// Numerics ("fast mode", tolerance-checked, NOT bit-exact): activations go through the reference's Q8_0
// quantisation (k_prep_q8_f16) and both operands are rounded to fp16 (<= 2^-11 relative each); products are exact
// in fp32 and accumulated in fp32 in hardware order.  Measured: 2.7e-4 relative RMS on one matmul; ~5e-3 per layer on
// hidden states, dominated by Q8_0 codes of the NEXT matmul's input flipping by one step (tests/test_gpu_fast_prefill.py).
#pragma once
#include "kernels.cuh"

namespace b200 {

constexpr int kFgM = 128, kFgN = 128, kFgK = 128;     // CTA tile: 128 weight rows x 128 tokens, K block of 128 (one quad)
constexpr int kFgStages = 2;
constexpr int kFgRawBytes = 4 * 4 * kQ4Chunk;         // 4 tiles x 4 row-groups x 576 B = one quad of 128 rows
constexpr int kFgABytes = kFgM * kFgK * 2;            // 32 KB: two [128 x 64] K-major SW128 sub-tiles
constexpr int kFgBBytes = kFgN * kFgK * 2;            // 32 KB
constexpr int kFgStageBytes = kFgRawBytes + kFgABytes + kFgBBytes;
constexpr int kFgSmem = kFgStages * kFgStageBytes + 1024 /*align*/ + 256;

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

struct FastGemmArgs {
    PackedW W;                  // G=1 packing for STORE/RESID (TR = 4), G=2 packing (TR = 8) for GATE
    const uint16_t * xh;        // [N][K] fp16 (k_prep_q8_f16)
    const float * resid; int ldr;
    float * y; int ldy;
    int N, out_rows;
    const uint16_t * tsilu;
};

template <int EPI>
__global__ void __launch_bounds__(160, 1) k_gemm_q4_tc(const FastGemmArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t * smem = (uint8_t *)(((uintptr_t) smem_raw + 1023) & ~(uintptr_t) 1023);       // SWIZZLE_128B tiles need 1 KB alignment
    uint64_t * bars = (uint64_t *)(smem + kFgStages * kFgStageBytes);
    uint64_t * raw_full = bars, * stage_free = bars + 2;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int mt = blockIdx.x, nt = blockIdx.y;             // 128-row tile, 128-token tile
    const int nbq = a.W.nbq, K = a.W.K;
    const int TRp = a.W.TR;                                 // row-groups per packed tile (4 or 8)
    const int tiles_per_m = 16 / TRp;                       // packed tiles per 128 rows (16 row-groups)

    if (tid == 0) {
        for (int s = 0; s < kFgStages; s++) { mbar_init(&raw_full[s], 1); mbar_init(&stage_free[s], 1); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 4) {
        if (lane == 0) {
            // ---------------------------------------------------------------- TMA producer (one thread)
            grid_dep_launch();
            for (int kb = 0; kb < nbq; kb++) {               // stream the raw quad of 128 rows for K block kb
                const int s = kb % kFgStages, use = kb / kFgStages;
                if (use > 0) mbar_wait(&stage_free[s], (use - 1) & 1);
                uint8_t * raw = smem + (size_t) s * kFgStageBytes;
                const uint32_t per_tile = (uint32_t) TRp * kQ4Chunk;
                mbar_arrive_expect_tx(&raw_full[s], (uint32_t) kFgRawBytes);
                for (int t = 0; t < tiles_per_m; t++) {
                    const uint8_t * src = a.W.data + (long long)(mt * tiles_per_m + t) * a.W.tile_bytes + (size_t) kb * per_tile;
                    bulk_g2s(raw + (size_t) t * per_tile, src, per_tile, &raw_full[s]);
                }
            }
        }
    } else {
        // -------------------------------------------------------------------- dequant + MMA warpgroup (128 threads)
        grid_dep_wait();
        float acc[2][64];                                    // rows 0..63 and 64..127 of the M tile
        #pragma unroll
        for (int h = 0; h < 2; h++)
            #pragma unroll
            for (int i = 0; i < 64; i++) acc[h][i] = 0.f;
        const int r8 = lane >> 2, w = lane & 3;
        for (int kb = 0; kb < nbq; kb++) {
            const int s = kb % kFgStages, use = kb / kFgStages;
            uint8_t * stage = smem + (size_t) s * kFgStageBytes;
            uint8_t * A = stage + kFgRawBytes, * B = A + kFgABytes;
            // B tile: tokens nt*128 .. +127, K block kb: [128 tokens][128 halfs] -> two SW128 sub-tiles (stage is free: the
            // wgmma group that last read it, K block kb-2, was retired by wgmma_wait<1> at the end of K block kb-1)
            mbar_wait(&raw_full[s], use & 1);
            for (int c = tid; c < kFgN * 16; c += 128) {     // 16-byte chunks: 128 rows x 16 chunks
                const int row = c >> 4, ch = c & 15, tok = nt * kFgN + row;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (tok < a.N && kb * kFgK + ch * 8 < K) v = *(const uint4 *)(a.xh + (size_t) tok * K + kb * kFgK + ch * 8);
                const int sub = ch >> 3, c8 = ch & 7;
                *(uint4 *)(B + sub * (kFgN * 128) + row * 128 + ((c8 ^ (row & 7)) << 4)) = v;
            }
            // A tile: this warp expands row-groups 4*warp .. 4*warp+3 (rows 32*warp .. +31) of the quad
            #pragma unroll
            for (int gi = 0; gi < 4; gi++) {
                const int g = warp * 4 + gi;                 // row-group 0..15 of the M tile, in packed order
                const uint8_t * ch = stage + (size_t) g * kQ4Chunk;
                const uint4 wv = *(const uint4 *)(ch + lane * 16);
                const uint2 sc = *(const uint2 *)(ch + 512 + r8 * 8);
                const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
                const uint32_t sw[2] = {sc.x, sc.y};
                const int row = g * 8 + r8;                  // row within the 128-row tile (packed order)
                #pragma unroll
                for (int bq = 0; bq < 4; bq++) {
                    const uint32_t x = ww[bq] ^ 0x88888888u;             // back to offset-binary nibbles n = v + 8
                    const uint32_t dh = (sw[bq >> 1] >> (16 * (bq & 1))) & 0xFFFFu;
                    const __half2 d2 = __halves2half2(__ushort_as_half((unsigned short) dh), __ushort_as_half((unsigned short) dh));
                    const __half2 off = __halves2half2(__ushort_as_half((unsigned short) 0x6408), __ushort_as_half((unsigned short) 0x6408));   // 1032.0
                    uint32_t h[4];                            // {e0,e2} {e16,e18} {e1,e3} {e17,e19} relative to 4w
                    #pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const uint32_t m = ((x >> (4 * i)) & 0x000F000Fu) | 0x64006400u;      // 1024 + n, exact in fp16
                        const __half2 v = __hmul2(__hsub2(*(const __half2 *) &m, off), d2);     // (n - 8) * d, one rounding
                        h[i] = *(const uint32_t *) &v;
                    }
                    // reorder pairs to consecutive k: lo = e0 e1 e2 e3, hi = e16 e17 e18 e19
                    const uint32_t lo0 = __byte_perm(h[0], h[2], 0x5410), lo1 = __byte_perm(h[0], h[2], 0x7632);
                    const uint32_t hi0 = __byte_perm(h[1], h[3], 0x5410), hi1 = __byte_perm(h[1], h[3], 0x7632);
                    const int klo = bq * 32 + 4 * w, khi = klo + 16;                      // k within the 128-wide block
                    {
                        const int sub = klo >> 6, kk = klo & 63, c8 = kk >> 3, within = (kk & 7) * 2;
                        *(uint2 *)(A + sub * (kFgM * 128) + row * 128 + ((c8 ^ (row & 7)) << 4) + within) = make_uint2(lo0, lo1);
                    }
                    {
                        const int sub = khi >> 6, kk = khi & 63, c8 = kk >> 3, within = (kk & 7) * 2;
                        *(uint2 *)(A + sub * (kFgM * 128) + row * 128 + ((c8 ^ (row & 7)) << 4) + within) = make_uint2(hi0, hi1);
                    }
                }
            }
            fence_proxy_async();                             // generic-proxy writes -> visible to the tensor core's async proxy
            named_bar_sync(1, 128);                          // A and B complete; the raw quad is consumed
            if (tid == 0) mbar_arrive(&stage_free[s]);
            const uint32_t a_addr = smem_u32(A), b_addr = smem_u32(B);
            wgmma_fence();
            acc_fence(acc[0]); acc_fence(acc[1]);
            #pragma unroll
            for (int k16 = 0; k16 < 8; k16++) {
                const uint32_t sub = (k16 >> 2) * (kFgM * 128), off = (k16 & 3) * 32;          // sub-tile of 64 K, 32 B per K step of 16
                #pragma unroll
                for (int h = 0; h < 2; h++)
                    wgmma_m64n128k16(acc[h], gmma_desc_k_sw128(a_addr + sub + h * (64 * 128) + off), gmma_desc_k_sw128(b_addr + sub + off));
            }
            wgmma_commit();
            wgmma_wait<1>();
            acc_fence(acc[0]); acc_fence(acc[1]);
        }
        wgmma_wait<0>();
        acc_fence(acc[0]); acc_fence(acc[1]);
        // -------------------------------------------------------------------- epilogue: registers -> global
        #pragma unroll
        for (int h = 0; h < 2; h++) gmma_epilogue<EPI>(a, acc[h], mt, h * 64 + warp * 16 + r8, nt * kFgN + 2 * w);
    }
}

}  // namespace b200
