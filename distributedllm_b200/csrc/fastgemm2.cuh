// fastgemm2.cuh -- K2, second generation: the prefill weight matmul as a wgmma tile kernel fed by TMA.
//
//   Y[token][row] = sum_k  W[row][k] * X[token][k]      W: Q4_0 or Q8_0 (packed layout of kernels.cuh), X: fp16 activations
//
// What changed against fastgemm.cuh:
//   * CTA tile 128 weight rows x 256 TOKENS (two consumer warpgroups, each 64 rows x 256 tokens as two wgmma m64n128k16
//     accumulators, 128 fp32 registers a thread): every dequantised weight tile is used against twice as many tokens;
//   * the activation tile comes in through the TENSOR-MAP TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B: the hardware writes
//     the K-major layout the GMMA descriptor expects), issued by the producer lane next to the 1-D bulk copy of the raw
//     quantised weights -- the dequant warps no longer spend half their instructions copying activations;
//   * 8 dequant warps instead of 4; each warpgroup dequantises its own 64 rows, issues their wgmma and keeps one K block in
//     flight while it dequantises the next, so dequantisation and tensor-core work overlap;
//   * Q8_0 weights as well as Q4_0 (int8 -> fp16 through the 0x6400 magic, one HMUL2 by the block scale).
// Numerics as fastgemm.cuh ("fast mode", tolerance-checked, NOT bit-exact): operands rounded to fp16, fp32 accumulation
// in hardware order.  Reference for the operation: ggml_compute_forward_mul_mat (ggml.c:10577-10749); the CUDA analogue in
// the reference tree is dequantise -> cublasSgemm (ggml-cuda.cu:2514-2560).
#pragma once
#include <cuda.h>

#include "fastgemm.cuh"

namespace b200 {

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
