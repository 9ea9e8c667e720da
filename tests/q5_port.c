/*
 * tests/q5_port.c -- TEST INFRASTRUCTURE.  Not product code.
 *
 * The Q5_0 / Q5_1 weight matmuls of the reference's AVX2+FMA+F16C build, restated in plain C on top of the slice
 * restatement in oracle/slice_oracle.c (included, not modified): every other operation of the forward -- Q8_0 / Q8_1
 * activation quantisation, RMSNorm, RoPE, the fp16 attention dots, softmax, SiLU -- is that file's, operand for operand.
 * tests/q5_port.py compiles this translation unit on first use; the GPU tests compare the Q5 kernels against it.
 *
 * Function            follows
 * ------------------  -------------------------------------------------------------
 * orc_dot_q5_0_q8_0   ggml_vec_dot_q5_0_q8_0, AVX2 branch (ggml.c:2914-2936): Q4_0's chain with a fifth bit per weight
 * orc_dot_q5_1_q8_1   ggml_vec_dot_q5_1_q8_1, AVX2 branch (ggml.c:3164-3189): Q4_1's chain with a fifth bit per weight
 * q5_forward          orc_forward (tensor_processor.cpp:537-766) with the Q5 matmul dispatch (vec_dot_type, ggml.c:1674-1681)
 * q5_logits           get_llm_output's RMSNorm + lm_head (tensor_processor.cpp:1850-1863) for any type q5_matmul takes
 */
#include "slice_oracle.c"

enum { W_Q5_0 = 6, W_Q5_1 = 7 };

/* element e of a Q5 block (qh = 4 bytes of fifth bits, qs = 16 nibble bytes): 0..31 (bytes_from_bits_32 + nibbles) */
static int q5_elem(const uint8_t * qh, const uint8_t * qs, int e) {
    const int n = e < 16 ? (qs[e] & 0x0F) : (qs[e - 16] >> 4);
    return n | (((qh[e >> 3] >> (e & 7)) & 1) << 4);
}

/* one row of Q5_0 blocks (22 B: fp16 d, u8 qh[4], 16 nibble bytes) . one Q8_0-quantised activation row.
 * Odd block counts are summed like even ones (the reference's assert(nb % 2 == 0) is compiled out by -DNDEBUG). */
float orc_dot_q5_0_q8_0(const uint8_t * w, const int8_t * aq, const uint16_t * ad, int k) {
    float acc[8] = {0};
    for (int b = 0; b < k / QK; b++) {
        const uint8_t * blk = w + (size_t) b * 22; uint16_t dw; memcpy(&dw, blk, 2);
        const float d = h2f(dw) * h2f(ad[b]);
        for (int l = 0; l < 8; l++) {
            int s = 0;
            for (int j = 0; j < 4; j++) s += (q5_elem(blk + 2, blk + 6, 4*l + j) - 16) * (int) aq[b*QK + 4*l + j];
            acc[l] = fmaf(d, (float) s, acc[l]);
        }
    }
    return hsum8(acc);
}

/* one row of Q5_1 blocks (24 B: fp16 d, fp16 m, u8 qh[4], 16 nibble bytes) . one Q8_1-quantised activation row */
float orc_dot_q5_1_q8_1(const uint8_t * w, const int8_t * aq, const float * ad, const float * as, int k) {
    float acc[8] = {0};
    float summs = 0.0f;
    for (int b = 0; b < k / QK; b++) {
        const uint8_t * blk = w + (size_t) b * 24; uint16_t dw, mw; memcpy(&dw, blk, 2); memcpy(&mw, blk + 2, 2);
        const float d = h2f(dw) * ad[b];
        summs += h2f(mw) * as[b];                      /* two roundings: -std=c11 builds do not contract */
        for (int l = 0; l < 8; l++) {
            int s = 0;
            for (int j = 0; j < 4; j++) s += q5_elem(blk + 4, blk + 8, 4*l + j) * (int) aq[b*QK + 4*l + j];
            acc[l] = fmaf((float) s, d, acc[l]);
        }
    }
    return hsum8(acc) + summs;
}

/* y[N][rows] = W[rows][k] . x[N][k]: Q5_0 with Q8_0 activations, Q5_1 with Q8_1; every other type as slice_oracle.c */
static void q5_matmul(const orc_slice * s, const uint8_t * W, int rows, int k, const float * x, int N, float * y) {
    const int nb = k / QK;
    if (s->wtype == W_Q5_0) {
        int8_t * aq = malloc((size_t) N * k); uint16_t * ad = malloc((size_t) N * nb * 2);
        for (int n = 0; n < N; n++) orc_quant_q8_0(x + (size_t) n * k, k, aq + (size_t) n * k, ad + (size_t) n * nb);
        const size_t rb = (size_t) nb * 22;
        #pragma omp parallel for schedule(static)
        for (int r = 0; r < rows; r++)
            for (int n = 0; n < N; n++)
                y[(size_t) n * rows + r] = orc_dot_q5_0_q8_0(W + r * rb, aq + (size_t) n * k, ad + (size_t) n * nb, k);
        free(aq); free(ad);
    } else if (s->wtype == W_Q5_1) {
        int8_t * aq = malloc((size_t) N * k); float * ad = malloc((size_t) N * nb * 4), * as = malloc((size_t) N * nb * 4);
        for (int n = 0; n < N; n++) orc_quant_q8_1(x + (size_t) n * k, k, aq + (size_t) n * k, ad + (size_t) n * nb, as + (size_t) n * nb);
        const size_t rb = (size_t) nb * 24;
        #pragma omp parallel for schedule(static)
        for (int r = 0; r < rows; r++)
            for (int n = 0; n < N; n++)
                y[(size_t) n * rows + r] = orc_dot_q5_1_q8_1(W + r * rb, aq + (size_t) n * k, ad + (size_t) n * nb, as + (size_t) n * nb, k);
        free(aq); free(ad); free(as);
    } else {
        matmul(s, W, rows, k, x, N, y);
    }
}

/* lm_head of an extra-layers file whose output.weight is Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 or F16 (wtype): RMSNorm * norm
 * weight, then y[N][n_vocab] = W . x as the layers' matmuls compute it */
void q5_logits(int wtype, const uint8_t * W, int n_vocab, int E, const float * norm_w, const float * x, int N, float * y) {
    init_tables();
    orc_slice s; memset(&s, 0, sizeof s); s.wtype = wtype;
    float * cur = malloc((size_t) N * E * 4);
    for (int n = 0; n < N; n++) orc_rmsnorm(x + (size_t) n * E, norm_w, E, cur + (size_t) n * E);
    q5_matmul(&s, W, n_vocab, E, cur, N, y);
    free(cur);
}

/* orc_forward with q5_matmul.  in/out: [N][n_embd] f32.  Returns 0, or 1 when the context would overflow. */
int q5_forward(orc_slice * s, const float * in, int N, float * out) {
    const int E = s->n_embd, H = s->n_head, D = E / H, FF = s->n_ff, n_past = s->n_past, T = n_past + N;
    if (T > s->n_ctx || N <= 0) return 1;
    float * x   = malloc((size_t) N * E * 4);   memcpy(x, in, (size_t) N * E * 4);
    float * cur = malloc((size_t) N * E * 4), * q = malloc((size_t) N * E * 4), * k = malloc((size_t) N * E * 4);
    float * v   = malloc((size_t) N * E * 4), * att = malloc((size_t) N * E * 4), * ffin = malloc((size_t) N * E * 4);
    float * g1  = malloc((size_t) N * FF * 4), * g3 = malloc((size_t) N * FF * 4);
    const float kq_scale = 1.0f / sqrtf((float) E / H);
    for (int il = 0; il < s->n_layer; il++) {
        const orc_layer * L = &s->layers[il];
        uint16_t * Kc = s->k + (size_t) il * s->n_ctx * E, * Vc = s->v + (size_t) il * s->n_ctx * E;
        for (int n = 0; n < N; n++) orc_rmsnorm(x + (size_t) n * E, L->attn_norm, E, cur + (size_t) n * E);
        q5_matmul(s, L->wk, E, E, cur, N, k);
        q5_matmul(s, L->wq, E, E, cur, N, q);
        q5_matmul(s, L->wv, E, E, cur, N, v);
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
            uint16_t qh[512]; float * sc = malloc((size_t) T * 4); uint16_t * ph = malloc((size_t) T * 2);
            for (int d = 0; d < D; d++) qh[d] = f2h(q[(size_t) n * E + h * D + d]);
            for (int t = 0; t < T; t++) {
                float kq = orc_dot_f16(Kc + (size_t) t * E + h * D, 1, qh, 1, D) * kq_scale;
                sc[t] = t > n_past + n ? -INFINITY : kq;
            }
            orc_softmax_row(sc, T);
            for (int t = 0; t < T; t++) ph[t] = f2h(sc[t]);
            for (int c = 0; c < D; c++) att[(size_t) n * E + h * D + c] = orc_dot_f16(Vc + h * D + c, E, ph, 1, T);
            free(sc); free(ph);
        }
        q5_matmul(s, L->wo, E, E, att, N, cur);
        for (size_t i = 0; i < (size_t) N * E; i++) ffin[i] = cur[i] + x[i];
        for (int n = 0; n < N; n++) orc_rmsnorm(ffin + (size_t) n * E, L->ffn_norm, E, cur + (size_t) n * E);
        q5_matmul(s, L->w3, FF, E, cur, N, g3);
        q5_matmul(s, L->w1, FF, E, cur, N, g1);
        for (size_t i = 0; i < (size_t) N * FF; i++) g1[i] = h2f(T_SILU[f2h(g1[i])]) * g3[i];
        q5_matmul(s, L->w2, E, FF, g1, N, cur);
        for (size_t i = 0; i < (size_t) N * E; i++) x[i] = cur[i] + ffin[i];
    }
    memcpy(out, x, (size_t) N * E * 4);
    s->n_past = T;
    free(x); free(cur); free(q); free(k); free(v); free(att); free(ffin); free(g1); free(g3);
    return 0;
}
