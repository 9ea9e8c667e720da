/*
 * oracle/slice_oracle.c -- TEST INFRASTRUCTURE.  Not product code.
 *
 * A plain-C restatement of the reference's per-slice forward: the arithmetic that
 * distllm/tensor_processor.cpp:474-809 (llama_eval_internal) asks vendor/llama.cpp/ggml.c
 * to perform, in the x86 AVX2+FMA+F16C build the reference's Makefile produces.  Every
 * rounding point and every accumulation order of that build is reproduced, so hidden
 * states are BIT-IDENTICAL to the compiled reference (pinned by tests/test_oracle.py against
 * tests/golden/*.npz, which gen_golden.py dumped from oracle/_ref = the reference itself).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this.
 *
 * Function            follows
 * ------------------  -------------------------------------------------------------
 * orc_fp32_to_fp16    GGML_FP32_TO_FP16 = _cvtss_sh(x, 0) (ggml.c:307-312): IEEE RNE
 * orc_quant_q8_0      quantize_row_q8_0, AVX branch (ggml.c:1215-1252)
 * orc_dot_q4_0_q8_0   ggml_vec_dot_q4_0_q8_0, AVX2 branch (ggml.c:2432-2455) + hsum_float_8 (614-620)
 * orc_dot_q8_0_q8_0   ggml_vec_dot_q8_0_q8_0, AVX2 branch (ggml.c:3313-3335)
 * orc_quant_q8_1      quantize_row_q8_1, AVX2 branch (ggml.c:1426-1484): d stays f32, s = d * sum(q)
 * orc_dot_q4_1_q8_1   ggml_vec_dot_q4_1_q8_1, AVX2 branch (ggml.c:2700-2733): the min term is a scalar float chain
 * orc_dot_f16         ggml_vec_dot_f16 (ggml.c:2323-2357) with GGML_F32x8_REDUCE (1895-1913)
 * orc_rmsnorm         ggml_compute_forward_rms_norm_f32 (ggml.c:10309-10352) + ggml_mul (9062)
 * orc_rope            ggml_compute_forward_rope_f32, mode 0 (ggml.c:11956-12055)
 * orc_softmax_row     ggml_compute_forward_soft_max_f32 (ggml.c:11524-11590), table_exp_f16 (4300-4312)
 * silu                ggml_vec_silu_f32 with GGML_SILU_FP16 (ggml.c:3541-3560), table 4310
 * orc_forward         tensor_processor.cpp:537-766 (one layer) and 1523-1544 (n_past bookkeeping)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define QK 32
enum { W_F32 = 0, W_F16 = 1, W_Q4_0 = 2, W_Q4_1 = 3, W_Q8_0 = 8 };

/* ---------------------------------------------------------------- fp16 <-> fp32 (software, IEEE RNE) */
static float h2f(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000) << 16, e = (h >> 10) & 0x1F, m = h & 0x3FF, u;
    if (e == 0) {
        if (m == 0) u = sign;
        else { int s = 0; while (!(m & 0x400)) { m <<= 1; s++; } m &= 0x3FF; u = sign | ((uint32_t)(113 - s) << 23) | (m << 13); }
    } else if (e == 31) u = sign | 0x7F800000u | (m << 13);
    else u = sign | ((e + 112) << 23) | (m << 13);
    float f; memcpy(&f, &u, 4); return f;
}
static uint16_t f2h(float f) {
    uint32_t u; memcpy(&u, &f, 4);
    uint32_t sign = (u >> 16) & 0x8000, a = u & 0x7FFFFFFFu;
    if (a >= 0x7F800000u) return (uint16_t)(sign | 0x7C00 | (a > 0x7F800000u ? 0x200 | ((a >> 13) & 0x3FF) : 0));
    if (a >= 0x477FF000u) return (uint16_t)(sign | 0x7C00);              /* rounds to inf */
    if (a < 0x33000001u) return (uint16_t)sign;                          /* < 2^-25 (or == 2^-25: ties to even 0) */
    int e = (int)(a >> 23) - 127; uint32_t m = (a & 0x7FFFFFu) | 0x800000u;
    int shift = e < -14 ? (13 + (-14 - e)) : 13;                         /* bits dropped */
    uint32_t q = m >> shift, rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (q & 1))) q++;
    uint32_t h = e < -14 ? q : (((uint32_t)(e + 15) << 10) + (q - 0x400));  /* carry propagates into exponent */
    return (uint16_t)(sign | h);
}
float    orc_fp16_to_fp32(uint16_t h) { return h2f(h); }
uint16_t orc_fp32_to_fp16(float f)    { return f2h(f); }

/* ---------------------------------------------------------------- lookup tables (ggml.c:4300-4312) */
static uint16_t T_EXP[65536], T_SILU[65536];
static int tables_ready = 0;
static void init_tables(void) {
    if (tables_ready) return;
    for (int i = 0; i < 65536; i++) {
        float f = h2f((uint16_t)i);
        T_EXP[i]  = f2h(expf(f));
        T_SILU[i] = f2h(f / (1.0f + expf(-f)));
    }
    tables_ready = 1;
}
void orc_tables(uint16_t * texp, uint16_t * tsilu) {
    init_tables(); memcpy(texp, T_EXP, sizeof T_EXP); memcpy(tsilu, T_SILU, sizeof T_SILU);
}

/* ---------------------------------------------------------------- activation quantisation */
/* x[k] -> q[k] int8, d[k/32] as fp16 bits */
void orc_quant_q8_0(const float * x, int k, int8_t * q, uint16_t * d) {
    for (int b = 0; b < k / QK; b++) {
        float amax = 0.0f;
        for (int j = 0; j < QK; j++) { float a = fabsf(x[b*QK + j]); if (a > amax) amax = a; }
        d[b] = f2h(amax / 127.f);
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        for (int j = 0; j < QK; j++) q[b*QK + j] = (int8_t) lrintf(x[b*QK + j] * id);   /* RNE (default rounding mode) */
    }
}

/* Q8_1: the block scale is NOT rounded to fp16, and s = d * (sum of the 32 quants) rides along for Q4_1's min term */
void orc_quant_q8_1(const float * x, int k, int8_t * q, float * d, float * s) {
    for (int b = 0; b < k / QK; b++) {
        float amax = 0.0f;
        for (int j = 0; j < QK; j++) { float a = fabsf(x[b*QK + j]); if (a > amax) amax = a; }
        d[b] = amax / 127.f;
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        int sum = 0;
        for (int j = 0; j < QK; j++) { q[b*QK + j] = (int8_t) lrintf(x[b*QK + j] * id); sum += q[b*QK + j]; }
        s[b] = d[b] * (float) sum;
    }
}

static float hsum8(const float a[8]) {            /* hsum_float_8, ggml.c:614-620 */
    float r0 = a[4] + a[0], r1 = a[5] + a[1], r2 = a[6] + a[2], r3 = a[7] + a[3];
    r0 = r0 + r2; r1 = r1 + r3;
    return r0 + r1;
}

/* one row of Q4_0 blocks (18 B each) . one Q8_0-quantised activation row */
float orc_dot_q4_0_q8_0(const uint8_t * w, const int8_t * aq, const uint16_t * ad, int k) {
    float acc[8] = {0};
    for (int b = 0; b < k / QK; b++) {
        const uint8_t * blk = w + (size_t) b * 18; uint16_t dw; memcpy(&dw, blk, 2);
        const float d = h2f(dw) * h2f(ad[b]);
        for (int l = 0; l < 8; l++) {
            int s = 0;
            for (int j = 0; j < 4; j++) {
                int e = 4*l + j;
                int wv = e < 16 ? (blk[2 + e] & 0x0F) : (blk[2 + e - 16] >> 4);
                s += (wv - 8) * (int) aq[b*QK + e];
            }
            acc[l] = fmaf(d, (float) s, acc[l]);
        }
    }
    return hsum8(acc);
}

/* one row of Q4_1 blocks (20 B: fp16 d, fp16 m, 16 nibble bytes) . one Q8_1-quantised activation row */
float orc_dot_q4_1_q8_1(const uint8_t * w, const int8_t * aq, const float * ad, const float * as, int k) {
    float acc[8] = {0};
    float summs = 0.0f;
    for (int b = 0; b < k / QK; b++) {
        const uint8_t * blk = w + (size_t) b * 20; uint16_t dw, mw; memcpy(&dw, blk, 2); memcpy(&mw, blk + 2, 2);
        const float d = h2f(dw) * ad[b];
        summs += h2f(mw) * as[b];                      /* two roundings: -std=c11 builds do not contract */
        for (int l = 0; l < 8; l++) {
            int s = 0;
            for (int j = 0; j < 4; j++) {
                int e = 4*l + j;
                int wv = e < 16 ? (blk[4 + e] & 0x0F) : (blk[4 + e - 16] >> 4);
                s += wv * (int) aq[b*QK + e];
            }
            acc[l] = fmaf(d, (float) s, acc[l]);
        }
    }
    return hsum8(acc) + summs;
}

float orc_dot_q8_0_q8_0(const uint8_t * w, const int8_t * aq, const uint16_t * ad, int k) {
    float acc[8] = {0};
    for (int b = 0; b < k / QK; b++) {
        const uint8_t * blk = w + (size_t) b * 34; uint16_t dw; memcpy(&dw, blk, 2);
        const float d = h2f(dw) * h2f(ad[b]);
        const int8_t * wq = (const int8_t *)(blk + 2);
        for (int l = 0; l < 8; l++) {
            int s = 0;
            for (int j = 0; j < 4; j++) s += (int) wq[4*l + j] * (int) aq[b*QK + 4*l + j];
            acc[l] = fmaf(d, (float) s, acc[l]);
        }
    }
    return hsum8(acc);
}

/* h2f of every fp16 bit pattern, for the inner loop below: the same values without the branches, which keeps the
 * attention over contexts of tens of thousands of positions affordable */
static float T_H2F[65536];
__attribute__((constructor)) static void init_h2f_table(void) {
    for (int i = 0; i < 65536; i++) T_H2F[i] = h2f((uint16_t) i);
}

/* x, y: fp16 bit patterns; y may be strided (V rows are walked over positions) */
float orc_dot_f16(const uint16_t * x, long xs, const uint16_t * y, long ys, int n) {
    const int np = n & ~31;
    float acc[32] = {0};
    for (int i = 0; i < np; i += 32)
        for (int s = 0; s < 32; s++) acc[s] = fmaf(T_H2F[x[(long)(i + s) * xs]], T_H2F[y[(long)(i + s) * ys]], acc[s]);
    float v[8];
    for (int l = 0; l < 8; l++) {                 /* x0+=x2; x1+=x3; x0+=x1 (GGML_F32x8_REDUCE, ARR=4) */
        float a0 = acc[l] + acc[16 + l], a1 = acc[8 + l] + acc[24 + l];
        v[l] = a0 + a1;
    }
    float t0 = v[0] + v[4], t1 = v[1] + v[5], t2 = v[2] + v[6], t3 = v[3] + v[7];
    double sumf = (double)((t0 + t1) + (t2 + t3));
    for (int i = np; i < n; i++) sumf += (double)(h2f(x[(long) i * xs]) * h2f(y[(long) i * ys]));
    return (float) sumf;
}

/* F32 weights: ggml_vec_dot_f32 (ggml.c:2170-2208) has the same 32-slot shape, no fp16 rounding */
static float dot_f32(const float * x, const float * y, int n) {
    const int np = n & ~31;
    float acc[32] = {0};
    for (int i = 0; i < np; i += 32) for (int s = 0; s < 32; s++) acc[s] = fmaf(x[i + s], y[i + s], acc[s]);
    float v[8];
    for (int l = 0; l < 8; l++) { float a0 = acc[l] + acc[16 + l], a1 = acc[8 + l] + acc[24 + l]; v[l] = a0 + a1; }
    float t0 = v[0] + v[4], t1 = v[1] + v[5], t2 = v[2] + v[6], t3 = v[3] + v[7];
    double sumf = (double)((t0 + t1) + (t2 + t3));
    for (int i = np; i < n; i++) sumf += (double)(x[i] * y[i]);
    return (float) sumf;
}

void orc_rmsnorm(const float * x, const float * w, int n, float * y) {
    double sum = 0.0;
    for (int i = 0; i < n; i++) sum += (double)(x[i] * x[i]);
    const float mean = (float)(sum / n);
    const float scale = 1.0f / sqrtf(mean + 1e-6f);
    for (int i = 0; i < n; i++) { float t = x[i] * scale; y[i] = w ? t * w[i] : t; }
}

/* x: [n_head][d_head] in place, position p */
void orc_rope(float * x, int n_head, int d_head, int p) {
    const float theta_scale = powf(10000.0, -2.0f / d_head);
    for (int h = 0; h < n_head; h++) {
        float theta = (float) p;
        for (int i0 = 0; i0 < d_head; i0 += 2) {
            const float c = cosf(theta), s = sinf(theta);
            theta *= theta_scale;
            float * v = x + h * d_head + i0;
            const float x0 = v[0], x1 = v[1];
            v[0] = x0*c - x1*s;
            v[1] = x0*s + x1*c;
        }
    }
}

void orc_softmax_row(float * p, int n) {
    init_tables();
    float mx = -INFINITY;
    for (int i = 0; i < n; i++) if (p[i] > mx) mx = p[i];
    double sum = 0.0;
    for (int i = 0; i < n; i++) {
        if (p[i] == -INFINITY) p[i] = 0.0f;
        else { float v = h2f(T_EXP[f2h(p[i] - mx)]); sum += (double) v; p[i] = v; }
    }
    const float inv = (float)(1.0 / sum);
    for (int i = 0; i < n; i++) p[i] *= inv;
}

float orc_silu(float x) { init_tables(); return h2f(T_SILU[f2h(x)]); }

/* ---------------------------------------------------------------- the slice */
typedef struct {
    const float * attn_norm, * ffn_norm;
    const uint8_t * wq, * wk, * wv, * wo, * w1, * w2, * w3;
} orc_layer;

typedef struct {
    int n_embd, n_head, n_ff, n_layer, n_ctx, wtype, n_past;
    orc_layer * layers;
    uint16_t * k, * v;          /* [n_layer][n_ctx][n_embd] fp16 bits */
} orc_slice;

orc_slice * orc_create(int n_embd, int n_head, int n_ff, int n_layer, int n_ctx, int wtype) {
    init_tables();
    orc_slice * s = calloc(1, sizeof *s);
    s->n_embd = n_embd; s->n_head = n_head; s->n_ff = n_ff; s->n_layer = n_layer; s->n_ctx = n_ctx; s->wtype = wtype;
    s->layers = calloc(n_layer, sizeof(orc_layer));
    s->k = calloc((size_t) n_layer * n_ctx * n_embd, 2);
    s->v = calloc((size_t) n_layer * n_ctx * n_embd, 2);
    return s;
}
void orc_set_layer(orc_slice * s, int il, const float * attn_norm, const void * wq, const void * wk, const void * wv,
                   const void * wo, const float * ffn_norm, const void * w1, const void * w2, const void * w3) {
    orc_layer * L = &s->layers[il];
    L->attn_norm = attn_norm; L->ffn_norm = ffn_norm;
    L->wq = wq; L->wk = wk; L->wv = wv; L->wo = wo; L->w1 = w1; L->w2 = w2; L->w3 = w3;
}
void orc_clear(orc_slice * s) {
    s->n_past = 0;
    memset(s->k, 0, (size_t) s->n_layer * s->n_ctx * s->n_embd * 2);
    memset(s->v, 0, (size_t) s->n_layer * s->n_ctx * s->n_embd * 2);
}
int  orc_n_past(orc_slice * s) { return s->n_past; }
void orc_set_n_past(orc_slice * s, int p) { s->n_past = p; }
void orc_free(orc_slice * s) { free(s->layers); free(s->k); free(s->v); free(s); }

/* y[N][rows] = W[rows][k] . x[N][k]   (ggml_compute_forward_mul_mat, ggml.c:10577-10749) */
static void matmul(const orc_slice * s, const uint8_t * W, int rows, int k, const float * x, int N, float * y) {
    const int nb = k / QK;
    if (s->wtype == W_Q4_0 || s->wtype == W_Q8_0) {
        int8_t * aq = malloc((size_t) N * k); uint16_t * ad = malloc((size_t) N * nb * 2);
        for (int n = 0; n < N; n++) orc_quant_q8_0(x + (size_t) n * k, k, aq + (size_t) n * k, ad + (size_t) n * nb);
        const size_t rb = (size_t) nb * (s->wtype == W_Q4_0 ? 18 : 34);
        #pragma omp parallel for schedule(static)
        for (int r = 0; r < rows; r++)
            for (int n = 0; n < N; n++)
                y[(size_t) n * rows + r] = s->wtype == W_Q4_0
                    ? orc_dot_q4_0_q8_0(W + r * rb, aq + (size_t) n * k, ad + (size_t) n * nb, k)
                    : orc_dot_q8_0_q8_0(W + r * rb, aq + (size_t) n * k, ad + (size_t) n * nb, k);
        free(aq); free(ad);
    } else if (s->wtype == W_Q4_1) {
        int8_t * aq = malloc((size_t) N * k); float * ad = malloc((size_t) N * nb * 4), * as = malloc((size_t) N * nb * 4);
        for (int n = 0; n < N; n++) orc_quant_q8_1(x + (size_t) n * k, k, aq + (size_t) n * k, ad + (size_t) n * nb, as + (size_t) n * nb);
        const size_t rb = (size_t) nb * 20;
        #pragma omp parallel for schedule(static)
        for (int r = 0; r < rows; r++)
            for (int n = 0; n < N; n++)
                y[(size_t) n * rows + r] = orc_dot_q4_1_q8_1(W + r * rb, aq + (size_t) n * k, ad + (size_t) n * nb, as + (size_t) n * nb, k);
        free(aq); free(ad); free(as);
    } else if (s->wtype == W_F16) {
        uint16_t * xh = malloc((size_t) N * k * 2);
        for (size_t i = 0; i < (size_t) N * k; i++) xh[i] = f2h(x[i]);
        #pragma omp parallel for schedule(static)
        for (int r = 0; r < rows; r++)
            for (int n = 0; n < N; n++)
                y[(size_t) n * rows + r] = orc_dot_f16((const uint16_t *) W + (size_t) r * k, 1, xh + (size_t) n * k, 1, k);
        free(xh);
    } else {
        #pragma omp parallel for schedule(static)
        for (int r = 0; r < rows; r++)
            for (int n = 0; n < N; n++)
                y[(size_t) n * rows + r] = dot_f32((const float *) W + (size_t) r * k, x + (size_t) n * k, k);
    }
}

/* in/out: [N][n_embd] f32.  Returns 0, or 1 when the context would overflow. */
int orc_forward(orc_slice * s, const float * in, int N, float * out) {
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
        matmul(s, L->wk, E, E, cur, N, k);
        matmul(s, L->wq, E, E, cur, N, q);
        matmul(s, L->wv, E, E, cur, N, v);
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
            /* score rows on the heap: n_ctx is a load parameter and reaches tens of thousands of positions */
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
        matmul(s, L->wo, E, E, att, N, cur);
        for (size_t i = 0; i < (size_t) N * E; i++) ffin[i] = cur[i] + x[i];
        for (int n = 0; n < N; n++) orc_rmsnorm(ffin + (size_t) n * E, L->ffn_norm, E, cur + (size_t) n * E);
        matmul(s, L->w3, FF, E, cur, N, g3);
        matmul(s, L->w1, FF, E, cur, N, g1);
        for (size_t i = 0; i < (size_t) N * FF; i++) g1[i] = h2f(T_SILU[f2h(g1[i])]) * g3[i];
        matmul(s, L->w2, E, FF, g1, N, cur);
        for (size_t i = 0; i < (size_t) N * E; i++) x[i] = cur[i] + ffin[i];
    }
    memcpy(out, x, (size_t) N * E * 4);
    s->n_past = T;
    free(x); free(cur); free(q); free(k); free(v); free(att); free(ffin); free(g1); free(g3);
    return 0;
}
