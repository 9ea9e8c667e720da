// kquant.cuh -- Q4_K / Q6_K layer matrices ("k-quants", QK_K = 256), exact mode.
//
// Restates the reference's AVX2+FMA build operand for operand, so hidden states are bit-identical:
//   act-quant   quantize_row_q8_K_reference        k_quants.c:1133-1168
//   Q4_K . Q8_K ggml_vec_dot_q4_K_q8_K, AVX2       k_quants.c:2450-2513
//   Q6_K . Q8_K ggml_vec_dot_q6_K_q8_K, AVX2       k_quants.c:3484-3561
//   embeddings  dequantize_row_q4_K                k_quants.c:733-756
// Both weight types take Q8_K activations (ggml.c:1710-1729): a matrix of either type that reads the same input sees the
// same quants.  An AVX lane l covers bytes 4l..4l+3 of every 32-byte vector; its int32 sum over a super-block is exact,
// then acc_l = fma(d, (float) sumi_l, acc_l) once per super-block and the row result is hsum_float_8(acc).
//   Q4_K: sumi_l = sum_j sc[2j] * (low nibbles . q8) + sc[2j+1] * (high nibbles . q8) over the 4 groups j of 32 bytes,
//         d = y.d * fp16(x.d); min term acc_m[i] = fma(-y.d * fp16(x.dmin), (float)(m[2i] q8s[2i] + m[2i+1] q8s[2i+1]),
//         acc_m[i]) with q8s[k] = the sum of sub-block k's 32 quants; result hsum_float_8(acc) + ((m0 + m2) + (m1 + m3)).
//   Q6_K: sumi_l = sum_{j<2, k<4} sc[8j + 2k + (l >= 4)] * ((q6 - 32) . q8); result hsum_float_8(acc).
// A Q6_K output.weight (the client-side lm_head) is packed and multiplied like the layers' Q6_K matrices.
#pragma once
#include "kernels.cuh"

namespace b200 {

// =============================================================================================
// Packed layout.  A chunk = 8 rows x ONE super-block, the file's bytes and nothing added; tiles as for the 32-wide types
// (kernels.cuh): tile t = [sb = 0..nbq) [rg = 0..TR) [chunk], nbq = super-blocks padded to a multiple of kKQS.
// Thread (r, w) = lane 4r + w of a consumer warp owns AVX lanes w and w+4 of row r.  What it reads of a 32-byte vector is
// bytes 4w..4w+3 ("lo") and 16+4w..16+4w+3 ("hi"); every 512-B plane holds 16 B per lane at lane * 16 (one conflict-free
// LDS.128).
// Q4_K chunk (1152 B = 8 x 144):
//      0 plane A : {group 0 lo, group 0 hi, group 1 lo, group 1 hi} of qs (group j = qs bytes 32j..32j+31)
//    512 plane B : the same for groups 2, 3
//   1024 header  : 16 B per row = the file's d, dmin, scales[12]
// Q6_K chunk (1680 B = 8 x 210):
//      0 plane A : {ql 0..31 lo, hi, ql 32..63 lo, hi}           (half j = 0)
//    512 plane B : {ql 64..95 lo, hi, ql 96..127 lo, hi}         (half j = 1)
//   1024 plane C : {qh 0..31 lo, hi, qh 32..63 lo, hi}
//   1536 scales  : 16 int8 per row
//   1664 d       : fp16 per row
// =============================================================================================
constexpr int kWT_Q4_K = 12;
constexpr int kQ4KChunk = 1152, kQ6KChunk = 1680;
constexpr int kKQS = 2;                 // super-blocks per ring stage (the Q4_K stage carries Q4_0's 9216 B)
static_assert(kQ4KChunk == 8 * 144 && kQ6KChunk == 8 * 210, "a chunk holds the file's bytes, nothing added");
static_assert(kQ4KChunk % 16 == 0 && kQ6KChunk % 16 == 0, "a ring stage stays one bulk copy");

__host__ __device__ constexpr bool wt_kquant(int wt) { return wt == kWT_Q4_K || wt == kWT_Q6_K; }
__host__ __device__ constexpr int kq_chunk_bytes(int wt) { return wt == kWT_Q4_K ? kQ4KChunk : kQ6KChunk; }
__host__ __device__ constexpr int kq_block_bytes(int wt) { return wt == kWT_Q4_K ? 144 : 210; }

// ---- repack: raw GGJT super-blocks -> packed chunks (one thread per output 32-bit word); modes as k_repack
__global__ void k_repack_kq(RepackArgs a) {
    const int cb = kq_chunk_bytes(a.wtype), words = cb / 4, bsz = kq_block_bytes(a.wtype);
    const bool q6 = a.wtype == kWT_Q6_K;
    const long long total = (long long) a.n_tiles * a.nbq * a.TR * words;
    for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < total; i += (long long) gridDim.x * blockDim.x) {
        const int wi = (int)(i % words);
        long long c = i / words;
        const int rg = (int)(c % a.TR); c /= a.TR;
        const int sb = (int)(c % a.nbq);
        const int tile = (int)(c / a.nbq);
        const int gi = tile * a.TR + rg;
        int s, sg;
        if (a.mode == 1)      { const int gps = a.rows_per_src / 8; s = gi / gps; sg = gi % gps; }
        else if (a.mode == 2) { s = gi & 1; sg = gi >> 1; }
        else                  { s = 0; sg = gi; }
        int r, off;                                          // row in the group, byte offset in the file's block
        if (wi < 384 && (q6 || wi < 256)) {                  // planes: lane L = 4r + w, component comp of its 16 B
            const int p = wi >> 7, lw = wi & 127, lane = lw >> 2, comp = lw & 3, w = lane & 3;
            r = lane >> 2;
            const int v32 = 2 * p + (comp >> 1);             // which 32-byte vector of the plane's 64 source bytes
            off = (q6 ? (p < 2 ? 64 * p + 32 * (comp >> 1) : 128 + 32 * (comp >> 1)) : 16 + 32 * v32) + 16 * (comp & 1) + 4 * w;
        } else if (!q6) {                                    // Q4_K header: d, dmin, scales[12]
            r = (wi - 256) >> 2; off = 4 * ((wi - 256) & 3);
        } else if (wi < 416) {                               // Q6_K scales
            r = (wi - 384) >> 2; off = 192 + 4 * ((wi - 384) & 3);
        } else {                                             // Q6_K d: rows 2t, 2t+1
            r = 2 * (wi - 416); off = 208;
        }
        uint32_t out = 0;
        const bool src_ok = s < 3 && a.src[s] != nullptr;
        const int row = sg * 8 + r;
        if (q6 && wi >= 416) {
            for (int k = 0; k < 2; k++)
                if (src_ok && row + k < a.rows_per_src && sb < a.nb)
                    out |= (uint32_t) *(const uint16_t *)(a.src[s] + ((long long)(row + k) * a.nb + sb) * bsz + off) << (16 * k);
        } else if (src_ok && row < a.rows_per_src && sb < a.nb) {
            const uint16_t * p = (const uint16_t *)(a.src[s] + ((long long) row * a.nb + sb) * bsz + off);
            out = (uint32_t) p[0] | ((uint32_t) p[1] << 16);
        }
        ((uint32_t *) a.dst)[i] = out;
    }
}

// ---- Q8_K act-quant of one super-block by one warp (quantize_row_q8_K_reference), written in the layout the matmul reads:
// per super-block 64 words [w][k = 2 * sub-block + (hi)], sub-block sums as[0..7], scale ad (f32, 1 / iscale).
// Lane L holds elements 8L..8L+7.  nw: RMSNorm weight (v = x * scale * nw, two roundings) or null.
__device__ __forceinline__ void warp_quant_q8k(const float * xs, const float * nw, float scale, int lane, int * aq, float * ad, int * as) {
    float v[8];
    const float4 t0 = *(const float4 *)(xs + lane * 8), t1 = *(const float4 *)(xs + lane * 8 + 4);
    v[0] = t0.x; v[1] = t0.y; v[2] = t0.z; v[3] = t0.w; v[4] = t1.x; v[5] = t1.y; v[6] = t1.z; v[7] = t1.w;
    if (nw) {
        const float4 w0 = __ldg((const float4 *)(nw + lane * 8)), w1 = __ldg((const float4 *)(nw + lane * 8 + 4));
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        #pragma unroll
        for (int j = 0; j < 8; j++) v[j] = fmul(fmul(v[j], scale), wv[j]);
    }
    // the FIRST element of the largest magnitude (`if (ax > amax)` in index order): key = (|v| bits, reversed index).
    // A NaN never passes `ax > amax`, so it is never the maximum, and a block of NaNs and zeros is a zero block (an
    // attention row whose scores are all NaN, from K cached as fp16 inf, reaches wo that way).
    uint32_t babs = 0; float best = 0.f; int bj = 0;
    #pragma unroll
    for (int j = 0; j < 8; j++) { const uint32_t u = __float_as_uint(fabsf(v[j])); if (u > babs && u <= 0x7F800000u) { babs = u; best = v[j]; bj = j; } }
    unsigned long long key = babs ? ((unsigned long long) babs << 32) | (unsigned)(255 - (lane * 8 + bj)) : 0ull;
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long k2 = __shfl_xor_sync(0xffffffffu, key, o); key = k2 > key ? k2 : key; }
    const int sbk = lane >> 2, b0 = 8 * (lane & 3), w0 = (b0 & 15) >> 2, kk = 2 * sbk + (b0 >> 4);
    if (key == 0ull) {                                       // all-zero block: d = 0, q = 0
        aq[w0 * 16 + kk] = 0; aq[(w0 + 1) * 16 + kk] = 0;
        if ((lane & 3) == 0) as[sbk] = 0;
        if (lane == 0) *ad = 0.f;
        return;
    }
    const int arg = 255 - (int)(key & 0xFFFFFFFFu);
    const float mx = __shfl_sync(0xffffffffu, best, arg >> 3);
    const float iscale = __fdiv_rn(-128.f, mx);
    uint32_t pk[2] = {0u, 0u}; int sum = 0;
    #pragma unroll
    for (int j = 0; j < 8; j++) {
        const float val = fadd(fmul(iscale, v[j]), 12582912.f);                       // nearest_int (k_quants.c:50-55)
        // nearest_int of a NaN reads the mantissa of x86's default NaN (0x400000): 0.  The GPU's NaN has mantissa 0x7FFFFF.
        const int q = val != val ? 0 : min(127, (int)((__float_as_uint(val) & 0x007fffffu) - 0x00400000));
        sum += q;
        pk[j >> 2] |= ((uint32_t)(q & 0xFF)) << (8 * (j & 3));
    }
    aq[w0 * 16 + kk] = (int) pk[0]; aq[(w0 + 1) * 16 + kk] = (int) pk[1];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    if ((lane & 3) == 0) as[sbk] = sum;
    if (lane == 0) *ad = __fdiv_rn(1.0f, iscale);
}

// the f32 scale plane of a column is padded to a multiple of 4 super-blocks, so every plane of a pre-quantised input
// (k_quant_q8k) is a whole number of 16-byte units and arrives by one bulk copy
__host__ __device__ constexpr int kq_nbd(int nbq) { return (nbq + 3) & ~3; }
__host__ __device__ inline size_t kq_act_bytes(int nbq, int NC) { return (size_t) NC * nbq * (256 + 32) + (size_t) NC * kq_nbd(nbq) * 4; }

// ---- Q8_K act-quant of whole rows in front of every k-quant matmul: [RMSNorm * weight ->] Q8_K once per token, in the
// shared-memory layout of k_gemv_kq, which fetches its columns with three bulk copies (PRO_PREQ).  Planes: aq [N][nbq*64] words, sums at aq + soff [N][nbq*8],
// scales ad [N][kq_nbd(nbq)].
struct QuantKArgs {
    const float * x; int ldx; const float * norm_w; int K;
    int * aq; int soff; float * ad; int nbq;
};

template <bool NORM>
__global__ void __launch_bounds__(256) k_quant_q8k(const QuantKArgs a) {
    __shared__ double red[8];
    const int n = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nb = a.K / 256;
    if (tid == 0) grid_dep_launch();
    grid_dep_wait();
    const float * x = a.x + (size_t) n * a.ldx;
    float scale = 1.0f;
    if (NORM) {                                        // ggml_compute_forward_rms_norm_f32 (sum in double)
        double s = 0.0;
        for (int i = tid * 4; i < a.K; i += 256 * 4) {
            const float4 v = *(const float4 *)(x + i);
            s += widen_nonneg(fmul(v.x, v.x)); s += widen_nonneg(fmul(v.y, v.y));
            s += widen_nonneg(fmul(v.z, v.z)); s += widen_nonneg(fmul(v.w, v.w));
        }
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[warp] = s;
        __syncthreads();
        const double tot = ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7]));
        scale = rms_scale(tot, x, a.K);
    }
    int * aq = a.aq + (size_t) n * a.nbq * 64;
    int * as = a.aq + a.soff + (size_t) n * a.nbq * 8;
    float * ad = a.ad + (size_t) n * kq_nbd(a.nbq);
    for (int sb = warp; sb < nb; sb += 8)
        warp_quant_q8k(x + sb * 256, NORM ? a.norm_w + sb * 256 : nullptr, scale, lane, aq + sb * 64, ad + sb, as + sb * 8);
}

// =============================================================================================
// K1k: Q4_K / Q6_K matmul.  The structure of k_gemv (producer warp + TMA ring from before griddepcontrol.wait, PDL trigger
// after the last weight copy, 4 consumer warps x 8 rows x G groups, NC columns, ring-less variant) with:
//   * prologue (PRO_PREQ only): k_quant_q8k, launched right before, quantised every input column once; three bulk copies
//     fetch the NC columns' quants, sub-block sums and scales.  A Q8_K block spans 256 outputs of the previous matmul,
//     more than any of its CTAs produces, so no producer epilogue can quantise it.  Quantising inside every CTA instead
//     (a bulk copy of the f32 row, [RMSNorm ->] Q8_K per super-block) measured 4-7 % slower on 7B decode and
//     re-quantised every column group of a prompt, so that variant is gone.
//   * epilogues: store | + residual (| send to the next rank) | SiLU(w1 x) * (w3 x).
// =============================================================================================
template <int WT, int G, int NC, int PRO, int EPI, bool RING>
__global__ void __launch_bounds__(kConsumers + 32) k_gemv_kq(const GemvArgs a) {
    static_assert(wt_kquant(WT), "k-quant weight type");
    static_assert(PRO == PRO_PREQ, "k-quant matmuls read inputs quantised by k_quant_q8k");
    static_assert(EPI == EPI_STORE || EPI == EPI_RESID || EPI == EPI_GATE || EPI == EPI_RESID_SEND, "k-quant epilogues");
    constexpr bool Q4K = WT == kWT_Q4_K;
    constexpr int CB = kq_chunk_bytes(WT);
    constexpr int TR = kWPC * G;
    constexpr int stage_bytes = kKQS * TR * CB;
    extern __shared__ __align__(128) uint8_t smem[];
    const int nbq = a.W.nbq, nb = a.W.nb, nbd = kq_nbd(nbq);
    const int NS = a.NS;
    // smem: [ring NS*stage][aq NC*nbq*256][as NC*nbq*8 int][ad NC*nbd f32][full 16][empty 16][act bar 2]
    uint8_t * ring = smem;
    int * aq_s = (int *)(smem + (RING ? (size_t) NS * stage_bytes : 0));
    int * as_s = aq_s + (size_t) NC * nbq * 64;
    float * ad_s = (float *)(as_s + (size_t) NC * nbq * 8);
    uint64_t * full = (uint64_t *)(ad_s + (size_t) NC * nbd);
    uint64_t * empty = full + 16;
    uint64_t * actbar = empty + 16;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int col0 = blockIdx.y * NC;
    const int n_stage = nbq / kKQS;

    if (tid == 0) {
        B200_TRACE(a.trace, 0);
        if (RING) for (int s = 0; s < NS; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], kWPC); }
        mbar_init(actbar, 1);
        mbar_init(actbar + 1, kWPC);        // gate: consumers have issued their prologue loads
        mbar_fence_init();
    }
    __syncthreads();

    if (RING && warp == kWPC) {
        // ------------------------------------------------------------------ producer warp (as k_gemv)
        if (lane == 0) {
            int slot = 0, use = 0, issued = 0;
            for (int tile = blockIdx.x; tile < a.W.n_tiles; tile += gridDim.x) {
                const uint8_t * src = a.W.data + (long long) tile * a.W.tile_bytes;
                for (int s = 0; s < n_stage; s++) {
                    if (issued == a.pre_stages) mbar_wait(actbar + 1, 0);
                    issued++;
                    if (use > 0) mbar_wait(&empty[slot], (use - 1) & 1);
                    mbar_arrive_expect_tx(&full[slot], (uint32_t) stage_bytes);
                    bulk_g2s(ring + (size_t) slot * stage_bytes, src + (size_t) s * stage_bytes, (uint32_t) stage_bytes, &full[slot]);
                    if (++slot == NS) { slot = 0; use++; }
                }
            }
            // the same ordering guarantee as k_gemv: never before the consumers returned from griddepcontrol.wait
            if (issued <= a.pre_stages) mbar_wait(actbar + 1, 0);
            grid_dep_launch();
            B200_TRACE(a.trace, 4);
        }
        return;
    }

    // ---------------------------------------------------------------------- consumer warps
    grid_dep_wait();                                   // the input comes from the previous kernel
    if (!RING && tid == 0) grid_dep_launch();
    if (tid == 0) B200_TRACE(a.trace, 1);

    const int ncols = min(NC, a.N - col0);
    // the input was quantised by k_quant_q8k; in_soff: words between the quant plane and the sub-block-sum plane of aq_in
    if (tid == 0) {
        const uint32_t b1 = (uint32_t) ncols * nbq * 256, b2 = (uint32_t) ncols * nbq * 32, b3 = (uint32_t) ncols * nbd * 4;
        mbar_arrive_expect_tx(actbar, b1 + b2 + b3);
        bulk_g2s(aq_s, a.aq_in + (size_t) col0 * nbq * 64, b1, actbar);
        bulk_g2s(as_s, a.aq_in + a.in_soff + (size_t) col0 * nbq * 8, b2, actbar);
        bulk_g2s(ad_s, a.da_in + (size_t) col0 * nbd, b3, actbar);
    }
    if (RING && lane == 0) mbar_arrive(actbar + 1);
    for (int n = ncols; n < NC; n++) {                 // padded columns: zeros
        for (int i = tid; i < nbq * 64; i += kConsumers) aq_s[(size_t) n * nbq * 64 + i] = 0;
        for (int i = tid; i < nbq * 8; i += kConsumers) as_s[(size_t) n * nbq * 8 + i] = 0;
        for (int i = tid; i < nbd; i += kConsumers) ad_s[(size_t) n * nbd + i] = 0.f;
    }
    mbar_wait(actbar, 0);
    named_bar_sync(1, kConsumers);                     // padded columns are zeroed by all warps
    if (tid == 0) B200_TRACE(a.trace, 2);

    const int r = lane >> 2, w = lane & 3;
    int slot = 0, phase = 0;
    uint2 * send_slot = nullptr; int send_seq = 0;
    if (EPI == EPI_RESID_SEND) {
        send_seq = a.mb_mine->seq_out + 1;
        if (lane == 0) mb_wait_slot_free(a.mb_mine, send_seq);
        __syncwarp();
        send_slot = a.mb_peer_inbox + (size_t)(send_seq & (kMbSlots - 1)) * a.mb_slot_elems;
    }
    for (int tile = blockIdx.x; tile < a.W.n_tiles; tile += gridDim.x) {
        float acc[G][NC][2], accm[G][NC];             // accm: Q4_K's min lane i = w (4 threads of a row = 4 lanes)
        #pragma unroll
        for (int g = 0; g < G; g++)
            #pragma unroll
            for (int n = 0; n < NC; n++) { acc[g][n][0] = 0.f; acc[g][n][1] = 0.f; accm[g][n] = 0.f; }
        const uint8_t * gsrc = a.W.data + (long long) tile * a.W.tile_bytes;

        for (int s = 0; s < n_stage; s++) {
            const uint8_t * base;
            if (RING) { mbar_wait(&full[slot], phase); base = ring + (size_t) slot * stage_bytes; }
            else base = gsrc + (size_t) s * stage_bytes;
            base += (size_t)(warp * G) * CB;
            if (!a.dbg_nomath)
            #pragma unroll
            for (int qi = 0; qi < kKQS; qi++) {
                const int sb = s * kKQS + qi;
                if (sb >= nb) break;                   // padding super-blocks are never summed
                uint4 pa[G], pb[G], pc[G], hd[G]; uint32_t dq[G];
                #pragma unroll
                for (int g = 0; g < G; g++) {
                    const uint8_t * ch = base + (size_t)(qi * TR + g) * CB;
                    pa[g] = *(const uint4 *)(ch + lane * 16);
                    pb[g] = *(const uint4 *)(ch + 512 + lane * 16);
                    if (Q4K) { hd[g] = *(const uint4 *)(ch + 1024 + r * 16); pc[g] = make_uint4(0u, 0u, 0u, 0u); dq[g] = 0u; }
                    else { pc[g] = *(const uint4 *)(ch + 1024 + lane * 16); hd[g] = *(const uint4 *)(ch + 1536 + r * 16);
                           dq[g] = *(const uint16_t *)(ch + 1664 + r * 2); }
                }
                #pragma unroll
                for (int n = 0; n < NC; n++) {
                    const int4 * ap = (const int4 *)(aq_s + (size_t) n * nbq * 64 + sb * 64 + w * 16);
                    const int4 a0 = ap[0], a1 = ap[1], a2 = ap[2], a3 = ap[3];
                    const int av[16] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
                    const float yd = ad_s[(size_t) n * nbd + sb];
                    int2 q8s = make_int2(0, 0);
                    if (Q4K) q8s = *(const int2 *)(as_s + (size_t) n * nbq * 8 + sb * 8 + 2 * w);
                    #pragma unroll
                    for (int g = 0; g < G; g++) {
                        int sumi[2] = {0, 0};
                        float d;
                        if (Q4K) {
                            // scales / mins (utmp, kmask1..3 of k_quants.c:2463-2468)
                            const uint32_t u0 = hd[g].y, u1 = hd[g].z, u2 = hd[g].w;
                            const uint32_t sc_lo = u0 & 0x3f3f3f3fu;
                            const uint32_t sc_hi = (u2 & 0x0f0f0f0fu) | (((u0 >> 6) & 0x03030303u) << 4);
                            const uint32_t mn_lo = u1 & 0x3f3f3f3fu;
                            const uint32_t mn_hi = ((u2 >> 4) & 0x0f0f0f0fu) | (((u1 >> 6) & 0x03030303u) << 4);
                            const uint32_t qw[8] = {pa[g].x, pa[g].y, pa[g].z, pa[g].w, pb[g].x, pb[g].y, pb[g].z, pb[g].w};
                            #pragma unroll
                            for (int j = 0; j < 4; j++) {
                                const uint32_t scw = j < 2 ? sc_lo : sc_hi;
                                const int s0 = (int)((scw >> (16 * (j & 1))) & 0xFF), s1 = (int)((scw >> (16 * (j & 1) + 8)) & 0xFF);
                                #pragma unroll
                                for (int h = 0; h < 2; h++) {
                                    const uint32_t q = qw[2 * j + h];
                                    sumi[h] += s0 * dp4a_us(q & 0x0F0F0F0Fu, av[2 * (2 * j) + h], 0)
                                             + s1 * dp4a_us((q >> 4) & 0x0F0F0F0Fu, av[2 * (2 * j + 1) + h], 0);
                                }
                            }
                            d = fmul(yd, h2f((uint16_t)(hd[g].x & 0xFFFFu)));
                            // min term, lane i = w: m[2w] * q8s[2w] + m[2w+1] * q8s[2w+1]
                            const uint32_t mw = w < 2 ? mn_lo : mn_hi;
                            const int m0 = (int)((mw >> (16 * (w & 1))) & 0xFF), m1 = (int)((mw >> (16 * (w & 1) + 8)) & 0xFF);
                            const float dmin = fmul(-yd, h2f((uint16_t)(hd[g].x >> 16)));
                            accm[g][n] = ffma(dmin, (float)(m0 * q8s.x + m1 * q8s.y), accm[g][n]);
                        } else {
                            const uint32_t sw[4] = {hd[g].x, hd[g].y, hd[g].z, hd[g].w};
                            const uint32_t l0[4] = {pa[g].x, pa[g].y, pa[g].z, pa[g].w};
                            const uint32_t l1[4] = {pb[g].x, pb[g].y, pb[g].z, pb[g].w};
                            const uint32_t qh[4] = {pc[g].x, pc[g].y, pc[g].z, pc[g].w};
                            #pragma unroll
                            for (int j = 0; j < 2; j++)
                                #pragma unroll
                                for (int k = 0; k < 4; k++) {
                                    const int sbi = 4 * j + k;
                                    #pragma unroll
                                    for (int h = 0; h < 2; h++) {
                                        const uint32_t ql = (j ? l1 : l0)[2 * (k & 1) + h];
                                        const uint32_t nib = (k & 2) ? (ql >> 4) & 0x0F0F0F0Fu : ql & 0x0F0F0F0Fu;
                                        const uint32_t q6 = nib | (((qh[2 * j + h] >> (2 * k)) & 0x03030303u) << 4);
                                        const int scv = (int)(int8_t)((sw[(2 * sbi + h) >> 2] >> (8 * ((2 * sbi + h) & 3))) & 0xFF);
                                        // (q6 ^ 32) << 2 = 4 * (q6 - 32) as signed bytes: the sum is 4x the lane's, exactly
                                        sumi[h] += scv * __dp4a((int)((q6 ^ 0x20202020u) << 2), av[2 * sbi + h], 0);
                                    }
                                }
                            sumi[0] >>= 2; sumi[1] >>= 2;
                            d = fmul(yd, h2f((uint16_t) dq[g]));
                        }
                        acc[g][n][0] = ffma(d, (float) sumi[0], acc[g][n][0]);
                        acc[g][n][1] = ffma(d, (float) sumi[1], acc[g][n][1]);
                    }
                }
            }
            if (RING) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[slot]);
                if (++slot == NS) { slot = 0; phase ^= 1; }
            }
        }

        // hsum_float_8 order ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)); Q4_K adds (m0+m2) + (m1+m3)
        float res[G][NC];
        #pragma unroll
        for (int g = 0; g < G; g++)
            #pragma unroll
            for (int n = 0; n < NC; n++) {
                float t = fadd(acc[g][n][0], acc[g][n][1]);
                t = fadd(t, __shfl_xor_sync(0xffffffffu, t, 2));
                t = fadd(t, __shfl_xor_sync(0xffffffffu, t, 1));
                if (Q4K) {
                    float m = fadd(accm[g][n], __shfl_xor_sync(0xffffffffu, accm[g][n], 2));
                    m = fadd(m, __shfl_xor_sync(0xffffffffu, m, 1));
                    t = fadd(t, m);
                }
                res[g][n] = t;
            }
        if (EPI == EPI_GATE) {
            const int row = (tile * kWPC + warp) * 8 + r;
            if (w == 0 && row < a.out_rows) {
                #pragma unroll
                for (int n = 0; n < NC; n++)
                    if (n < ncols) a.y[(size_t)(col0 + n) * a.ldy + row] = fmul(h2f(a.tsilu[f2h(res[0][n])]), res[G - 1][n]);
            }
        } else if (w == 0) {
            #pragma unroll
            for (int g = 0; g < G; g++) {
                const int row = ((tile * kWPC + warp) * G + g) * 8 + r;
                if (row < a.out_rows) {
                    #pragma unroll
                    for (int n = 0; n < NC; n++) {
                        if (n < ncols) {
                            float v = res[g][n];
                            if (EPI == EPI_RESID || EPI == EPI_RESID_SEND) v = fadd(v, a.resid[(size_t)(col0 + n) * a.ldr + row]);
                            a.y[(size_t)(col0 + n) * a.ldy + row] = v;
                            if (EPI == EPI_RESID_SEND) st_ll(send_slot + row, v, send_seq);
                        }
                    }
                }
            }
        }
    }
    if (tid == 0) B200_TRACE(a.trace, 3);
}

// dequantize_row_q4_K (k_quants.c:733-756): d1 * q - m1 with d1 = d * sc and m1 = min * m (no contraction: -std=c11)
__device__ __forceinline__ float dequant_q4k(const uint8_t * blk, int i) {
    const float d = h2f(*(const uint16_t *) blk), mn = h2f(*(const uint16_t *)(blk + 2));
    const uint8_t * q = blk + 4;                             // scales[12]
    const int j = i >> 5;                                    // sub-block (get_scale_min_k4)
    int sc, m;
    if (j < 4) { sc = q[j] & 63; m = q[j + 4] & 63; }
    else       { sc = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4); }
    const int byte = blk[16 + 32 * (j >> 1) + (i & 31)];
    const int qv = (j & 1) ? (byte >> 4) : (byte & 0xF);
    return fsub(fmul(fmul(d, (float) sc), (float) qv), fmul(mn, (float) m));
}

}  // namespace b200
