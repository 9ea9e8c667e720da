/*
 * tests/kq_port.c -- TEST INFRASTRUCTURE.  Not product code.
 *
 * The Q4_K / Q6_K weight matmuls of the reference's AVX2+FMA+F16C build (QK_K = 256), restated in plain C on top of the
 * slice restatement in oracle/slice_oracle.c (included, not modified): RMSNorm, RoPE, the fp16 attention dots, softmax
 * and SiLU are that file's, operand for operand.  A k-quant slice mixes types per matrix (Q4_K_M: wv / w2 are Q6_K in
 * some layers), so kq_forward takes the type of every matrix.
 *
 * Function              follows
 * --------------------  -------------------------------------------------------------
 * orc_quantize_q8_K     quantize_row_q8_K_reference (k_quants.c:1133-1168)
 * orc_dot_q4_K_q8_K     ggml_vec_dot_q4_K_q8_K, AVX2 branch (k_quants.c:2450-2513)
 * orc_dot_q6_K_q8_K     ggml_vec_dot_q6_K_q8_K, AVX2 branch (k_quants.c:3484-3561)
 * orc_dequant_q4_K      dequantize_row_q4_K (k_quants.c:733-756)
 * kq_forward            orc_forward (tensor_processor.cpp:537-766), each matrix dispatched on its own type
 *                       (vec_dot_type Q8_K for both, ggml.c:1710-1729)
 */
#include "slice_oracle.c"

#define QK_K 256
enum { W_Q4_K = 12, W_Q6_K = 14 };

/* x[k] -> q[k] int8, d[k/256] f32, bsums[k/16] (int16 in ggml; kept as int) */
void orc_quantize_q8_K(const float * x, int k, int8_t * q, float * d, int * bsums) {
    for (int i = 0; i < k / QK_K; i++, x += QK_K, q += QK_K) {
        float max = 0, amax = 0;
        for (int j = 0; j < QK_K; ++j) { const float ax = fabsf(x[j]); if (ax > amax) { amax = ax; max = x[j]; } }
        if (!amax) { d[i] = 0; memset(q, 0, QK_K); memset(bsums + 16 * i, 0, 16 * sizeof(int)); continue; }
        const float iscale = -128.f / max;
        for (int j = 0; j < QK_K; ++j) {
            const float val = iscale * x[j] + 12582912.f;       /* nearest_int (k_quants.c:50-55); -std=c11: no contraction */
            int iv; memcpy(&iv, &val, 4);
            const int v = (iv & 0x007fffff) - 0x00400000;
            q[j] = (int8_t)(v < 127 ? v : 127);
        }
        for (int j = 0; j < QK_K / 16; ++j) { int s = 0; for (int ii = 0; ii < 16; ++ii) s += q[j * 16 + ii]; bsums[16 * i + j] = s; }
        d[i] = 1 / iscale;
    }
}

/* get_scale_min_k4 (k_quants.c:593-601) */
static void scale_min_k4(int j, const uint8_t * q, int * sc, int * m) {
    if (j < 4) { *sc = q[j] & 63; *m = q[j + 4] & 63; }
    else { *sc = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); *m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4); }
}

/* one row of Q4_K super-blocks (144 B: fp16 d, fp16 dmin, scales[12], qs[128]) . one Q8_K row */
float orc_dot_q4_K_q8_K(const uint8_t * w, const int8_t * q8, const float * yd, const int * bsums, int k) {
    float acc[8] = {0}, acc_m[4] = {0};
    for (int i = 0; i < k / QK_K; i++) {
        const uint8_t * x = w + (size_t) i * 144; uint16_t dh, mh; memcpy(&dh, x, 2); memcpy(&mh, x + 2, 2);
        const float d = yd[i] * h2f(dh), dmin = -yd[i] * h2f(mh);
        int sc[8], m[8];
        for (int j = 0; j < 8; j++) scale_min_k4(j, x + 4, &sc[j], &m[j]);
        const int * bs = bsums + 16 * i;
        for (int l = 0; l < 4; l++) {                       /* madd(mins, hadd(bsums)) */
            const int prod = m[2*l] * (bs[4*l] + bs[4*l + 1]) + m[2*l + 1] * (bs[4*l + 2] + bs[4*l + 3]);
            acc_m[l] = fmaf(dmin, (float) prod, acc_m[l]);
        }
        const int8_t * y = q8 + (size_t) i * QK_K;
        for (int l = 0; l < 8; l++) {                       /* lane l: bytes 4l..4l+3 of each 32-byte group */
            int sumi = 0;
            for (int j = 0; j < 4; j++) {
                int lo = 0, hi = 0;
                for (int e = 0; e < 4; e++) {
                    const int b = x[16 + 32 * j + 4 * l + e];
                    lo += (b & 0xF) * y[64 * j + 4 * l + e];
                    hi += (b >> 4) * y[64 * j + 32 + 4 * l + e];
                }
                sumi += sc[2*j] * lo + sc[2*j + 1] * hi;
            }
            acc[l] = fmaf(d, (float) sumi, acc[l]);
        }
    }
    const float m02 = acc_m[0] + acc_m[2], m13 = acc_m[1] + acc_m[3];
    return hsum8(acc) + (m02 + m13);
}

/* one row of Q6_K super-blocks (210 B: ql[128], qh[64], int8 scales[16], fp16 d) . one Q8_K row */
float orc_dot_q6_K_q8_K(const uint8_t * w, const int8_t * q8, const float * yd, int k) {
    float acc[8] = {0};
    for (int i = 0; i < k / QK_K; i++) {
        const uint8_t * x = w + (size_t) i * 210; uint16_t dh; memcpy(&dh, x + 208, 2);
        const float d = yd[i] * h2f(dh);
        const int8_t * sc = (const int8_t *)(x + 192);
        const int8_t * y = q8 + (size_t) i * QK_K;
        for (int l = 0; l < 8; l++) {
            int sumi = 0;
            for (int j = 0; j < 2; j++)
                for (int kk = 0; kk < 4; kk++) {
                    int s = 0;
                    for (int e = 0; e < 4; e++) {
                        const int b = 4 * l + e;                     /* byte of the 32-byte vector */
                        const int ql = x[64 * j + 32 * (kk & 1) + b];
                        const int q6 = ((kk & 2 ? ql >> 4 : ql) & 0xF) | (((x[128 + 32 * j + b] >> (2 * kk)) & 3) << 4);
                        s += (q6 - 32) * y[128 * j + 32 * kk + b];
                    }
                    sumi += sc[8 * j + 2 * kk + (l >= 4)] * s;
                }
            acc[l] = fmaf(d, (float) sumi, acc[l]);
        }
    }
    return hsum8(acc);
}

/* tok_embeddings row of Q4_K super-blocks -> f32 */
void orc_dequant_q4_K(const uint8_t * w, int k, float * y) {
    for (int i = 0; i < k / QK_K; i++) {
        const uint8_t * x = w + (size_t) i * 144; uint16_t dh, mh; memcpy(&dh, x, 2); memcpy(&mh, x + 2, 2);
        const float d = h2f(dh), min = h2f(mh);
        for (int j = 0; j < 8; j++) {
            int sc, m; scale_min_k4(j, x + 4, &sc, &m);
            const float d1 = d * sc, m1 = min * m;
            for (int l = 0; l < 32; l++) {
                const int b = x[16 + 32 * (j >> 1) + l];
                *y++ = d1 * ((j & 1) ? b >> 4 : b & 0xF) - m1;
            }
        }
    }
}

/* y[N][rows] = W[rows][k] . x[N][k] for a Q4_K / Q6_K matrix */
static void kq_matmul(int type, const uint8_t * W, int rows, int k, const float * x, int N, float * y) {
    const int nb = k / QK_K;
    int8_t * q = malloc((size_t) N * k); float * d = malloc((size_t) N * nb * 4); int * bs = malloc((size_t) N * nb * 16 * sizeof(int));
    for (int n = 0; n < N; n++) orc_quantize_q8_K(x + (size_t) n * k, k, q + (size_t) n * k, d + (size_t) n * nb, bs + (size_t) n * nb * 16);
    const size_t rb = (size_t) nb * (type == W_Q4_K ? 144 : 210);
    #pragma omp parallel for schedule(static)
    for (int r = 0; r < rows; r++)
        for (int n = 0; n < N; n++)
            y[(size_t) n * rows + r] = type == W_Q4_K
                ? orc_dot_q4_K_q8_K(W + r * rb, q + (size_t) n * k, d + (size_t) n * nb, bs + (size_t) n * nb * 16, k)
                : orc_dot_q6_K_q8_K(W + r * rb, q + (size_t) n * k, d + (size_t) n * nb, k);
    free(q); free(d); free(bs);
}

/* orc_forward with kq_matmul.  types: [n_layer][wq, wk, wv, wo, w1, w2, w3].  in/out: [N][n_embd] f32.
 * Returns 0, or 1 when the context would overflow. */
int kq_forward(orc_slice * s, const int * types, const float * in, int N, float * out) {
    const int E = s->n_embd, H = s->n_head, D = E / H, FF = s->n_ff, n_past = s->n_past, T = n_past + N;
    if (T > s->n_ctx || N <= 0) return 1;
    float * x   = malloc((size_t) N * E * 4);   memcpy(x, in, (size_t) N * E * 4);
    float * cur = malloc((size_t) N * E * 4), * q = malloc((size_t) N * E * 4), * k = malloc((size_t) N * E * 4);
    float * v   = malloc((size_t) N * E * 4), * att = malloc((size_t) N * E * 4), * ffin = malloc((size_t) N * E * 4);
    float * g1  = malloc((size_t) N * FF * 4), * g3 = malloc((size_t) N * FF * 4);
    const float kq_scale = 1.0f / sqrtf((float) E / H);
    for (int il = 0; il < s->n_layer; il++) {
        const orc_layer * L = &s->layers[il];
        const int * t = types + 7 * il;
        uint16_t * Kc = s->k + (size_t) il * s->n_ctx * E, * Vc = s->v + (size_t) il * s->n_ctx * E;
        for (int n = 0; n < N; n++) orc_rmsnorm(x + (size_t) n * E, L->attn_norm, E, cur + (size_t) n * E);
        kq_matmul(t[1], L->wk, E, E, cur, N, k);
        kq_matmul(t[0], L->wq, E, E, cur, N, q);
        kq_matmul(t[2], L->wv, E, E, cur, N, v);
        for (int n = 0; n < N; n++) {
            orc_rope(k + (size_t) n * E, H, D, n_past + n);
            orc_rope(q + (size_t) n * E, H, D, n_past + n);
            for (int e = 0; e < E; e++) {
                Kc[(size_t)(n_past + n) * E + e] = f2h(k[(size_t) n * E + e]);
                Vc[(size_t)(n_past + n) * E + e] = f2h(v[(size_t) n * E + e]);
            }
        }
        #pragma omp parallel for schedule(static) collapse(2)
        for (int n = 0; n < N; n++) for (int h = 0; h < H; h++) {
            uint16_t qh[512]; float sc[8192]; uint16_t ph[8192];
            for (int d = 0; d < D; d++) qh[d] = f2h(q[(size_t) n * E + h * D + d]);
            for (int tt = 0; tt < T; tt++) {
                float kq = orc_dot_f16(Kc + (size_t) tt * E + h * D, 1, qh, 1, D) * kq_scale;
                sc[tt] = tt > n_past + n ? -INFINITY : kq;
            }
            orc_softmax_row(sc, T);
            for (int tt = 0; tt < T; tt++) ph[tt] = f2h(sc[tt]);
            for (int c = 0; c < D; c++) att[(size_t) n * E + h * D + c] = orc_dot_f16(Vc + h * D + c, E, ph, 1, T);
        }
        kq_matmul(t[3], L->wo, E, E, att, N, cur);
        for (size_t i = 0; i < (size_t) N * E; i++) ffin[i] = cur[i] + x[i];
        for (int n = 0; n < N; n++) orc_rmsnorm(ffin + (size_t) n * E, L->ffn_norm, E, cur + (size_t) n * E);
        kq_matmul(t[6], L->w3, FF, E, cur, N, g3);
        kq_matmul(t[4], L->w1, FF, E, cur, N, g1);
        for (size_t i = 0; i < (size_t) N * FF; i++) g1[i] = h2f(T_SILU[f2h(g1[i])]) * g3[i];
        kq_matmul(t[5], L->w2, E, FF, g1, N, cur);
        for (size_t i = 0; i < (size_t) N * E; i++) x[i] = cur[i] + ffin[i];
    }
    memcpy(out, x, (size_t) N * E * 4);
    s->n_past = T;
    free(x); free(cur); free(q); free(k); free(v); free(att); free(ffin); free(g1); free(g3);
    return 0;
}

/* lm_head of an extra-layers file with a Q6_K output.weight: RMSNorm * norm weight, then Q8_K . Q6_K per vocab row */
void kq_logits(const uint8_t * W, int n_vocab, int E, const float * norm_w, const float * x, int N, float * y) {
    init_tables();
    float * cur = malloc((size_t) N * E * 4);
    for (int n = 0; n < N; n++) orc_rmsnorm(x + (size_t) n * E, norm_w, E, cur + (size_t) n * E);
    kq_matmul(W_Q6_K, W, n_vocab, E, cur, N, y);
    free(cur);
}
