// runtime.cu -- slice handle, loader, forward scheduling and the C ABI (include/b200_slice.h).
//
// Replaces TransformerSlice / llama_eval_internal / the loader of the reference
// (distllm/tensor_processor.cpp:1488-1562, 474-809, 926-1086, 1203-1416) for a slice resident on
// one H100.  One stream per slice; the N=1 decode step is a CUDA graph replayed per token with
// the position kept in device memory.
#include "kernels.cuh"
#include "kquant.cuh"
#include "fastgemm2.cuh"
#include "kvstate.cuh"
#include "ggjt_file.hpp"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <cmath>
#include <condition_variable>
#include <dlfcn.h>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <type_traits>
#include <vector>

namespace b200 {

constexpr int kSmemLimit = 226 * 1024;   // opt-in dynamic limit is 227 KB minus static __shared__

struct LayerW {
    PackedW qkv{}, wo{}, w13{}, w2{};
    // k-quant slices: wq / wk / wv of different types are packed per run of one type (qkv holds the first run); the
    // other runs write rows qkv_row[i] onward of the same qkv output
    PackedW qkv_more[2]{}; int qkv_row[2] = {0, 0};
    // F16-weight slices
    uint16_t * f_q = nullptr, * f_k = nullptr, * f_v = nullptr, * f_o = nullptr, * f_1 = nullptr, * f_2 = nullptr, * f_3 = nullptr;
    float * attn_norm = nullptr, * ffn_norm = nullptr;
};

struct GraphKey { const float * in; float * out; int host; bool operator<(const GraphKey & o) const {
    return in != o.in ? in < o.in : (out != o.out ? out < o.out : host < o.host); } };

}  // namespace b200

using namespace b200;

struct b200_slice {
    int device = 0, n_sm = 132;
    cudaStream_t stream = nullptr;
    int E = 0, H = 0, D = 0, FF = 0, L = 0, first_layer = 0, n_ctx = 512, wtype = 0;
    // sessions (SURVEY 8f N3): independent sequences sharing the weights, each with its own KV cache and position.
    // Session 0 is the reference's single global context (tensor_processor.cpp:1491, 1992).
    int n_sessions = 1, cur = 0;
    std::vector<int> past;                 // n_past per session
    int * d_npast = nullptr;               // [n_sessions], device copy (graph replays read it)
    size_t sess_stride = 0;                // elements between two sessions' KV caches
    int * d_kvdst = nullptr;               // [n_sessions]: destination list of the last KV fan-out (k_kv_fanout)
    // batched and mixed passes (begin_pass): segment k runs segs[k].count tokens of session segs[k].session; the device table
    // d_pass holds, per pass, column -> (session, position), segment -> (session, count) and, when a segment has more than
    // one token, column -> row length (the end of its segment) and the tile table of the query-tiled attention
    struct Seg { int session, past, count, col; };
    std::vector<Seg> segs; std::vector<int> h_pass;
    int * d_pass = nullptr; const int2 * cols = nullptr; const int * col_T = nullptr; const int2 * d_segs = nullptr;
    const AttnTile * d_tiles = nullptr; int n_tiles = 0, tile_rows = 0;
    // decode rows (begin_steps): the pass is N single-token steps of one session, its table built on the device, and every
    // column attends with its own row length T = position + 1
    bool steps = false;
    std::vector<LayerW> layers;
    std::vector<void *> allocs;
    uint16_t * kc = nullptr, * vc = nullptr, * q16 = nullptr;
    float * xa = nullptr, * xb = nullptr, * qkv = nullptr, * att = nullptr, * ffin = nullptr, * gate = nullptr;
    float * d_in = nullptr, * d_out = nullptr, * h_in = nullptr, * h_out = nullptr;
    float2 * cs = nullptr; uint16_t * texp = nullptr, * tsilu = nullptr;
    int * aq_att = nullptr, * aq_gate = nullptr; float * da_att = nullptr, * da_gate = nullptr;   // pre-quantised activations
    int nbqE = 0, nbqF = 0;
    int soffE = 0, soffF = 0;              // Q4_1 slices (Q8_1 activations): floats between the scale plane and the block-sum plane of da_*
    int * aq_x = nullptr; float * da_x = nullptr; int * nq_counter = nullptr; double * nq_partial = nullptr;   // normalised+quantised layer input (last-CTA epilogue)
    std::map<GraphKey, cudaGraphExec_t> graphs;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr; bool timed = false;
    int64_t launches = 0, weight_bytes = 0;
    bool use_ring = true, use_graph = true, use_pdl = false, use_nq = true, f16_ring = true, use_tiled_attn = true, f16_mc = true; int f16_mc_cols = 4;
    bool skip_attention = false;   // measurement aid: replay only the weight matmuls of a step (bench.py roofline)
    bool attn_lut_smem = true;     // single-token attention stages the exp table in shared memory (decided at load)
    bool fast_prefill = false; int fast_min_tokens = 32; uint16_t * xh = nullptr;   // tensor-core prefill (fast mode)
    bool fast_pass = false;        // b200_perplexity_windows(fast = 1): mixed passes of any row count take fast mode too
    int opt_ns = 0, opt_cta_per_sm = 0, opt_nc = 0, opt_pre = 3, opt_nomath = 0;   // read once at load (environment)
    float ema_token_ms = 0.f;              // host-buffer decode calls: smoothed device time of one token (sleep-then-poll wait)
    std::mutex mu;
    // per-kernel-class event timing (b200_slice_profile): class 0 qkv, 1 rope, 2 attention, 3 wo, 4 w13, 5 w2, 6 advance
    bool profiling = false; int cur_class = 0;
    std::vector<cudaEvent_t> prof_ev; std::vector<int> prof_cls; size_t prof_used = 0;
    cudaEvent_t mark[2] = {nullptr, nullptr};
    // debug timeline
    unsigned long long * trace = nullptr; int trace_next = 0; std::vector<int> trace_cls, trace_ctas;
    // layer-slice pipeline over NCCL (see b200_pipeline_*)
    void * nccl_comm = nullptr; int pp_rank = 0, pp_world = 1; float * d_final = nullptr;
    // peer-memory hand-off (b200_pipeline_mailbox_*): my mailbox, and my ring neighbours' mailboxes mapped over NVLink
    uint8_t * mb_block = nullptr; size_t mb_slot_floats = 0;
    uint8_t * mb_next = nullptr, * mb_prev = nullptr; bool mb_on = false;
    bool send_pending = false; PeerSendArgs send_args{}; int send_ctas = 1;      // enqueue_layers launches the send right behind the last matmul
    // single-token steps fold the send into the slice's last matmul (EPI_RESID_SEND): rows leave for the next rank's inbox
    // as they are computed, no k_peer_send launch on the critical path
    bool fold_send = false, use_fold = true;
    // k-quant slices: the Q8_K input of the next matmul, quantised once per column (k_quant_q8k, PRO_PREQ)
    int * kq_aq = nullptr; float * kq_ad = nullptr;
    std::map<GraphKey, cudaGraphExec_t> pp_graphs;
    // the generation stream (b200_stream_open) this handle belongs to until b200_stream_close; every other entry point
    // refuses the handle meanwhile
    const b200_stream * owner = nullptr;
};

namespace b200 {

static int env_int(const char * name, int dflt) { const char * v = getenv(name); return v ? atoi(v) : dflt; }

template <typename T> static int dev_alloc(b200_slice * s, T ** p, size_t n) {
    void * q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T));
    if (e != cudaSuccess) return fail(B200_ECUDA, "cudaMalloc(%zu) failed: %s", n * sizeof(T), cudaGetErrorString(e));
    s->allocs.push_back(q); *p = (T *) q; return 0;
}

// ---------------------------------------------------------------- per-launch event brackets
static void prof_begin(b200_slice * s) {
    if (!s->profiling) return;
    if (s->prof_used + 2 > s->prof_ev.size()) {
        for (int i = 0; i < 2; i++) { cudaEvent_t e; cudaEventCreate(&e); s->prof_ev.push_back(e); }
    }
    cudaEventRecord(s->prof_ev[s->prof_used], s->stream);
}
static void prof_end(b200_slice * s) {
    if (!s->profiling) return;
    cudaEventRecord(s->prof_ev[s->prof_used + 1], s->stream);
    s->prof_cls.push_back(s->cur_class);
    s->prof_used += 2;
}

// ---------------------------------------------------------------- kernel launch
// Every kernel of a forward goes through here: programmatic dependent launch when enabled, the per-launch profile
// events and the launch count.
template <typename K, typename... A>
static int launch(b200_slice * s, K kern, dim3 grid, dim3 block, size_t smem, const A &... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = s->use_pdl ? 1 : 0;
    prof_begin(s);
    B200_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
    prof_end(s);
    s->launches++;
    return 0;
}

// A kernel's opt-in dynamic shared memory limit (with `carveout`, also the largest shared-memory carve-out), set once per
// device.  The flags are per kernel because every kernel is its own template argument (the k_gemv instantiations share
// one function type).
template <auto Kern>
static int smem_attr(const b200_slice * s, int bytes, bool carveout = false) {
    static bool done[16] = {false};
    if (done[s->device & 15]) return 0;
    B200_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (carveout) B200_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    done[s->device & 15] = true;
    return 0;
}

// Calls f(std::integral_constant<int, WT>{}) for weight type wt: one of the block-quantised types (Q4_0, Q4_1, Q5_0, Q5_1,
// Q8_0), or with KQ one of the k-quants (Q4_K, Q6_K).  Only the kernels of that family are instantiated (k_gemv_kq has no
// PRO_NORM prologue).  `what` names the missing kernel in the error.
template <bool KQ, class F>
static int with_wtype(int wt, const char * what, F && f) {
    using std::integral_constant;
    if constexpr (KQ) {
        switch (wt) {
        case kWT_Q4_K: return f(integral_constant<int, kWT_Q4_K>{});
        case kWT_Q6_K: return f(integral_constant<int, kWT_Q6_K>{});
        }
    } else {
        switch (wt) {
        case kWT_Q4_0: return f(integral_constant<int, kWT_Q4_0>{});
        case kWT_Q4_1: return f(integral_constant<int, kWT_Q4_1>{});
        case kWT_Q5_0: return f(integral_constant<int, kWT_Q5_0>{});
        case kWT_Q5_1: return f(integral_constant<int, kWT_Q5_1>{});
        case kWT_Q8_0: return f(integral_constant<int, kWT_Q8_0>{});
        }
    }
    return fail(B200_EINVAL, "no %s for weight type %d", what, wt);
}

// ---------------------------------------------------------------- weight matmuls
// Dynamic shared memory of a k_gemv launch: `act` bytes for the NC columns' activations (plus the f32 input row of a
// one-column PRO_NORM launch) and barriers, and `stage` bytes per ring stage; a launch with NS stages needs bytes(NS).
struct GemvSmem {
    size_t stage, act;
    size_t bytes(int NS) const { return (size_t) NS * stage + act; }
};

template <int WT, int G, int NC, int PRO>
static GemvSmem gemv_smem(const PackedW & W) {
    GemvSmem m;
    if constexpr (wt_kquant(WT)) {
        m.stage = (size_t) kKQS * kWPC * G * kq_chunk_bytes(WT);
        m.act = kq_act_bytes(W.nbq, NC) + 34 * 8 + 64;
        return m;
    }
    m.stage = (size_t) kQS * kWPC * G * chunk_bytes(WT);
    m.act = (size_t) NC * act_bytes_per_col(W.nbq, WT) + 34 * 8 + kWPC * 8 + (size_t) NC * 128 + 64 +
            ((NC == 1 && PRO == PRO_NORM) ? (size_t) W.K * 4 : 0);
    return m;
}

template <int WT, int G, int NC, int PRO, int EPI, bool RING>
static constexpr auto gemv_kernel() {
    if constexpr (wt_kquant(WT)) return k_gemv_kq<WT, G, NC, PRO, EPI, RING>;
    else return k_gemv<WT, G, NC, PRO, EPI, RING>;
}

template <int WT, int G, int NC, int PRO, int EPI, bool RING>
static int launch_gemv_t(b200_slice * s, GemvArgs a) {
    constexpr auto kern = gemv_kernel<WT, G, NC, PRO, EPI, RING>();
    const GemvSmem sm = gemv_smem<WT, G, NC, PRO>(a.W);
    const size_t stage = sm.stage, act = sm.act;
    // Ring depth: as deep as possible while EVERY tile of the matrix still gets a co-resident CTA (no second wave):
    // wide matrices (qkv 384 tiles, w1|w3 688) run 3-5 small-ring CTAs per SM, narrow ones (wo, w2: 128 tiles) one
    // CTA per SM with a deep ring.  B200_NS overrides.
    int NS = 0;
    if (RING) {
        const int ncolg = (a.N + NC - 1) / NC;
        int need = (a.W.n_tiles * ncolg + s->n_sm - 1) / s->n_sm;
        if (need > 5) need = 5;
        const size_t budget = (size_t) kSmemLimit / need - 1024;
        NS = s->opt_ns > 0 ? s->opt_ns : (budget > act ? (int)((budget - act) / stage) : 2);
        if (NS < 2) NS = 2;
        if (NS > 16) NS = 16;
        while (NS > 2 && NS * stage + act > (size_t) kSmemLimit) NS--;
    }
    const size_t smem = sm.bytes(NS);
    if (smem > (size_t) kSmemLimit) return fail(B200_EINVAL, "gemv needs %zu B of shared memory (K=%d, NC=%d)", smem, a.W.K, NC);
    // without the carve-out the driver's heuristic leaves room for only 2 CTAs/SM however small the ring is
    if (int rc = smem_attr<kern>(s, kSmemLimit, true)) return rc;
    a.NS = NS; a.dbg_nomath = s->opt_nomath; a.pre_stages = s->opt_pre;
    a.trace = nullptr;
    if (s->trace && s->trace_next < 512) { a.trace = s->trace + (size_t) s->trace_next * 1024 * 8; s->trace_next++; s->trace_cls.push_back(s->cur_class); }
    int per_sm = s->opt_cta_per_sm > 0 ? s->opt_cta_per_sm : (int)(kSmemLimit / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 6) per_sm = 6;
    const int ncol = (a.N + NC - 1) / NC;
    int gx = a.W.n_tiles;
    const int cap = s->n_sm * per_sm;
    if (gx > cap) gx = cap;
    if (a.trace) s->trace_ctas.push_back(gx * ncol);
    return launch(s, kern, dim3(gx, ncol, 1), dim3(RING ? kConsumers + 32 : kConsumers, 1, 1), smem, a);
}

template <int WT, int G, int PRO, int EPI>
static int launch_gemv_nc(b200_slice * s, const GemvArgs & a) {
    if (a.N == 1) return s->use_ring ? launch_gemv_t<WT, G, 1, PRO, EPI, true>(s, a) : launch_gemv_t<WT, G, 1, PRO, EPI, false>(s, a);
    if (!s->use_ring) return launch_gemv_t<WT, G, 8, PRO, EPI, false>(s, a);
    // Columns per CTA.  A multi-column step is issue-bound (every column repeats the dp4a -> fadd -> fma chains), so it
    // needs warps, not bytes: 8 columns per CTA amortise the nibble unpacking best, but a small batch (<= 8 columns)
    // over a narrow matrix (wo / w2: 128-160 tiles) would then run ONE 4-warp CTA per SM.  Take the widest column
    // group that still puts >= 3 CTAs on every SM; the extra column groups re-read the tile from L2, not from HBM
    // (they are co-resident and walk the tiles in the same order).
    // A group is taken only if its launch fits in shared memory with a two-stage ring: at LLaMA-65B (w2: K = 22016) eight
    // columns of activations plus two stages exceed it for Q8_0, Q4_1 and Q5_1 weights, whose w2 launches take four.
    // B200_NC forces a group, as an upper bound.
    const int want = 3 * s->n_sm, nt = a.W.n_tiles;
    const int force = s->opt_nc, cap = force > 0 ? force : 8;
    if (cap >= 8 && gemv_smem<WT, G, 8, PRO>(a.W).bytes(2) <= (size_t) kSmemLimit && (force || nt * ((a.N + 7) / 8) >= want))
        return launch_gemv_t<WT, G, 8, PRO, EPI, true>(s, a);
    if (cap >= 4 && gemv_smem<WT, G, 4, PRO>(a.W).bytes(2) <= (size_t) kSmemLimit && (force || nt * ((a.N + 3) / 4) >= want))
        return launch_gemv_t<WT, G, 4, PRO, EPI, true>(s, a);
    return launch_gemv_t<WT, G, 2, PRO, EPI, true>(s, a);
}

template <int G, int PRO, int EPI>
static int launch_gemv(b200_slice * s, const GemvArgs & a) {
    return with_wtype<false>(a.W.wtype, "block-quantised matmul",
                             [&](auto wt) { return launch_gemv_nc<decltype(wt)::value, G, PRO, EPI>(s, a); });
}

// Q4_K / Q6_K matrices (kquant.cuh): the type is per matrix, the activations are always Q8_K, quantised in the prologue
template <int G, int PRO, int EPI>
static int launch_gemv_kq(b200_slice * s, const GemvArgs & a) {
    return with_wtype<true>(a.W.wtype, "k-quant matmul",
                            [&](auto wt) { return launch_gemv_nc<decltype(wt)::value, G, PRO, EPI>(s, a); });
}

// The slice's last w2 of a single-token step with the pipeline send folded in (EPI_RESID_SEND): its rows leave for the
// next rank's inbox as they are computed.  One column, ring kernel.
template <bool KQ>
static int launch_w2_send(b200_slice * s, GemvArgs w) {
    w.mb_mine = (MailboxHdr *) s->mb_block;
    w.mb_peer_inbox = (uint2 *)(s->mb_next + sizeof(MailboxHdr)); w.mb_slot_elems = s->mb_slot_floats;
    return with_wtype<KQ>(w.W.wtype, "pipelined matmul",
                          [&](auto wt) { return launch_gemv_t<decltype(wt)::value, 1, 1, PRO_PREQ, EPI_RESID_SEND, true>(s, w); });
}

// The input of a k-quant matmul: [RMSNorm * norm_w ->] Q8_K of its N columns, once per column (k_quant_q8k), into the
// slice's Q8_K buffer, from which the matmul's CTAs fetch it (PRO_PREQ).
static int quant_kq(b200_slice * s, GemvArgs & a, bool norm) {
    const int nbq = a.W.nbq;
    QuantKArgs q{a.x, a.ldx, a.norm_w, a.W.K, s->kq_aq, s->n_ctx * nbq * 64, s->kq_ad, nbq};
    a.aq_in = s->kq_aq; a.in_soff = q.soff; a.da_in = s->kq_ad;
    return norm ? launch(s, k_quant_q8k<true>, dim3(a.N, 1, 1), dim3(256, 1, 1), 0, q)
                : launch(s, k_quant_q8k<false>, dim3(a.N, 1, 1), dim3(256, 1, 1), 0, q);
}

template <int PRO, int EPI>
static int launch_f16(b200_slice * s, GemvF16Args a) {
    int rc;
    if (a.N == 1 && s->use_ring && s->f16_ring && (a.K & 255) == 0) {
        // single-token steps: TMA-ring variant (weights stream from before the dependency wait, two CTAs per SM)
        if ((rc = smem_attr<k_gemv_f16_ring<PRO, EPI>>(s, kSmemLimit, true))) return rc;
        const int nc8 = (a.K / 32 + 7) / 8;
        const size_t fixed = (size_t) nc8 * 1024 + 64 + 64;
        int NS = s->opt_ns > 0 ? s->opt_ns : (int)(((size_t) 112 * 1024 - fixed) / ((size_t) kF16Warps * (kF16Stage + 16)));
        if (NS < 2) NS = 2;
        if (NS > 12) NS = 12;
        const size_t rsmem = (size_t) kF16Warps * NS * kF16Stage + (size_t) nc8 * 1024 + (size_t) 2 * kF16Warps * NS * 8 + 64;
        const int n_tiles = (a.rows + kF16Warps - 1) / kF16Warps;
        int per_sm = (int)(kSmemLimit / (rsmem + 1024)); if (per_sm < 1) per_sm = 1; if (per_sm > 4) per_sm = 4;
        int rgx = n_tiles < s->n_sm * per_sm ? n_tiles : s->n_sm * per_sm;
        return launch(s, k_gemv_f16_ring<PRO, EPI>, dim3(rgx, 1, 1), dim3(kF16Warps * 32 + 32, 1, 1), rsmem, a, NS);
    }
    if (a.N >= 2 && s->f16_mc) {
        // multi-token call: 8 (or 4) columns per CTA share every weight load (k_gemv_f16_mc)
        // 4 columns per CTA keep the activation block at 64 KB for K = 4096: three CTAs (24 warps) per SM; B200_F16_MC=8 forces 8
        const bool c8 = s->f16_mc_cols == 8 && a.N > 4 && (size_t) a.K * 4 * 8 + 64 <= (size_t) 200 * 1024;
        const int nc = c8 ? 8 : 4;
        const size_t msmem = (size_t) a.K * 4 * nc + 64;
        if (msmem <= (size_t) 72 * 1024 || (c8 && msmem <= (size_t) kSmemLimit)) {
            const int ncolg = (a.N + nc - 1) / nc;
            int per_sm = (int)(kSmemLimit / (msmem + 1024)); if (per_sm < 1) per_sm = 1;
            int mgx = (a.rows + 15) / 16;                    // 8 warps x 2 rows per CTA
            const int mcap = (s->n_sm * per_sm + ncolg - 1) / ncolg;
            if (mgx > mcap) mgx = mcap < 1 ? 1 : mcap;
            if (c8) {
                if ((rc = smem_attr<k_gemv_f16_mc<PRO, EPI, 8>>(s, kSmemLimit))) return rc;
                return launch(s, k_gemv_f16_mc<PRO, EPI, 8>, dim3(mgx, ncolg, 1), dim3(256, 1, 1), msmem, a);
            }
            if ((rc = smem_attr<k_gemv_f16_mc<PRO, EPI, 4>>(s, kSmemLimit))) return rc;
            return launch(s, k_gemv_f16_mc<PRO, EPI, 4>, dim3(mgx, ncolg, 1), dim3(256, 1, 1), msmem, a);
        }
    }
    int gx = (a.rows + 7) / 8;
    const int cap = s->n_sm * 8;
    if (gx > cap) gx = cap;
    if ((rc = smem_attr<k_gemv_f16<PRO, EPI>>(s, kSmemLimit))) return rc;
    return launch(s, k_gemv_f16<PRO, EPI>, dim3(gx, a.N, 1), dim3(256, 1, 1), (size_t) a.K * 2 + 16, a);
}

static int launch_norm_quant(b200_slice * s, const float * x, int ldx, const float * norm_w, int N) {
    NormQuantArgs q{x, ldx, norm_w, s->E, s->aq_x, s->da_x, s->nbqE, s->soffE};
    return with_wtype<false>(s->wtype, "activation quantiser", [&](auto wt) {
        return launch(s, k_norm_quant<decltype(wt)::value>, dim3(N, 1, 1), dim3(256, 1, 1), 0, q);
    });
}

// ---------------------------------------------------------------- fast-mode prefill (wgmma), see fastgemm2.cuh
template <bool NORM>
static int launch_prep(b200_slice * s, const float * x, int ldx, const float * norm_w, int K, int N) {
    PrepArgs p{x, ldx, norm_w, s->xh, K, N};
    return launch(s, k_prep_q8_f16<NORM>, dim3(N, 1, 1), dim3(256, 1, 1), 0, p);
}

// 128 x 256 (or 128 x 128) tiles, activations through a tensor-map TMA
typedef CUresult (*TensorMapEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                      const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TensorMapEncodeFn tensor_map_encode() {
    static TensorMapEncodeFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void * p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = (TensorMapEncodeFn) p;
    });
    return fn;
}

template <int WT, int EPI, int NT>
static int launch_fast_gemm_t(b200_slice * s, const PackedW & W, const float * resid, int ldr, float * y, int ldy, int N, int out_rows) {
    TensorMapEncodeFn enc = tensor_map_encode();
    if (!enc) return fail(B200_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    // activations xh [N][K] fp16, K innermost; box = 64 halfs (128 B, the swizzle span) x 256 token rows; rows >= N read as zeros
    CUtensorMap map;
    const cuuint64_t dims[2] = {(cuuint64_t) W.K, (cuuint64_t) N};
    const cuuint64_t strides[1] = {(cuuint64_t) W.K * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t) NT};
    const cuuint32_t estr[2] = {1, 1};
    CUresult cr = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *) s->xh, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return fail(B200_ECUDA, "cuTensorMapEncodeTiled failed (%d) for K=%d N=%d", (int) cr, W.K, N);
    if (int rc = smem_attr<k_gemm_tc2<WT, EPI, NT>>(s, f2_smem(WT, NT))) return rc;
    FastGemm2Args a{}; a.W = W; a.resid = resid; a.ldr = ldr; a.y = y; a.ldy = ldy; a.N = N; a.out_rows = out_rows; a.tsilu = s->tsilu;
    const int groups = W.n_tiles * W.TR;                     // 8-row groups in packed order
    return launch(s, k_gemm_tc2<WT, EPI, NT>, dim3((groups + 15) / 16, (N + NT - 1) / NT, 1), dim3(kF2Threads, 1, 1), f2_smem(WT, NT), a, map);
}

template <int EPI>
static int launch_fast_gemm(b200_slice * s, const PackedW & W, const float * resid, int ldr, float * y, int ldy, int N, int out_rows) {
    // 256-token tiles halve the dequantisation per flop; a matrix whose 128-row tiles x 256-token tiles would leave SMs idle
    // (wo, w2: 32 row tiles) takes 128-token tiles and three stages instead
    const int mtiles = (W.n_tiles * W.TR + 15) / 16;
    const bool wide = (long long) mtiles * ((N + 255) / 256) >= s->n_sm || N <= 128;
    if (W.wtype == kWT_Q4_0) return wide ? launch_fast_gemm_t<kWT_Q4_0, EPI, 256>(s, W, resid, ldr, y, ldy, N, out_rows)
                                         : launch_fast_gemm_t<kWT_Q4_0, EPI, 128>(s, W, resid, ldr, y, ldy, N, out_rows);
    return wide ? launch_fast_gemm_t<kWT_Q8_0, EPI, 256>(s, W, resid, ldr, y, ldy, N, out_rows)
                : launch_fast_gemm_t<kWT_Q8_0, EPI, 128>(s, W, resid, ldr, y, ldy, N, out_rows);
}

// ---------------------------------------------------------------- attention
// Dynamic shared memory of the attention kernels at this n_ctx: scores (f32) and probabilities (f16) of every position,
// then for head size 128 the staged K / V rows of the cluster kernel (up to 128 local rows = 512 positions) and in
// single-token steps the exp table's negative half, for other head sizes the partial sums of k_attention.
struct AttnSmem { int pf_rows; size_t plain, staged, lut, generic; };

static AttnSmem attn_smem(int n_ctx, int D) {
    AttnSmem m;
    const size_t sc = (size_t)((n_ctx + 3) & ~3) * 4 + (size_t)((n_ctx + 7) & ~7) * 2, sc16 = (sc + 15) & ~(size_t) 15;
    m.pf_rows = std::min(8 * ((n_ctx + 31) / 32), 128);
    m.plain = sc16 + 64;                                                   // k_attn128<false>
    m.staged = sc16 + (size_t) 2 * m.pf_rows * kAttnRow + 32 * 64 + 64;    // k_attn128<true>
    m.lut = m.staged + 65536;                                              // k_attn128<true>, exp table staged
    m.generic = sc + (size_t) 4 * D * 8 * 4 + 64;                          // k_attention
    return m;
}

// A prompt segment of a mixed pass whose whole context fits the staged window takes the query-tiled attention kernel
static bool seg_tiled(const b200_slice * s, const b200_slice::Seg & g) {
    return s->D == 128 && s->use_tiled_attn && g.count > 1 && g.past + g.count <= kAttnTMax;
}

// RoPE, KV-cache append and attention of layer il over s->qkv, into s->att.  With `preq` the head-size-128 kernels also
// write their output quantised for the wo matmul (aq_att / da_att).
static int attention(b200_slice * s, int il, int N, bool preq) {
    if (s->skip_attention) return 0;      // measurement aid: the matmul kernels of the step back to back
    const int E = s->E, H = s->H, D = s->D;
    // cols mode (batched independent sequences): the kernels add session * sess_stride themselves
    const size_t sess_off = s->cols ? 0 : (size_t) s->cur * s->sess_stride;
    uint16_t * kc = s->kc + sess_off + (size_t) il * s->n_ctx * E, * vc = s->vc + sess_off + (size_t) il * s->n_ctx * E;
    int * d_npast = s->d_npast + s->cur;
    const AttnSmem am = attn_smem(s->n_ctx, D);
    const float kq_scale = 1.0f / sqrtf((float) E / (float) H);
    int rc;
    if (D != 128) {
        s->cur_class = 1;
        RopeArgs ra{s->qkv, E, H, D, N, d_npast, s->cs, s->q16, kc, vc, s->cols, s->sess_stride};
        if ((rc = launch(s, k_rope_append, dim3((E / 2 + 255) / 256, N, 1), dim3(256, 1, 1), 0, ra))) return rc;
        s->cur_class = 2;
        AttnArgs aa{s->q16, kc, vc, d_npast, E, H, D, N, s->texp, s->att, kq_scale, s->cols, s->sess_stride, s->col_T};
        return launch(s, k_attention, dim3(H, N, 1), dim3(512, 1, 1), am.generic, aa);
    }
    // head size 128: cluster kernel; for single-token and batched steps RoPE + KV append are fused into its prologue
    constexpr int kChunk = 1024;     // query tokens per launch (grid.y)
    Attn128Args aa{};
    aa.pf_rows = am.pf_rows;
    aa.qkv = s->qkv; aa.q16 = s->q16; aa.kc = kc; aa.vc = vc; aa.n_past = d_npast; aa.E = E; aa.H = H; aa.N = N;
    aa.cols = s->cols; aa.sess_stride = s->sess_stride;
    aa.cs = s->cs; aa.texp = s->texp; aa.out = s->att;
    aa.n_ctx = s->n_ctx; aa.kq_scale = kq_scale;
    const float dsc = preq ? wt_act_scale(s->wtype) : 0.f;
    if (preq) { aa.aq_out = s->aq_att; aa.da_out = s->da_att; aa.out_nbq = s->nbqE; aa.out_dscale = dsc; aa.out_soff = s->soffE; }
    // the query-tiled kernel over a prompt chunk of one session (tiles null) or over every tile of a mixed pass; t_rows is the
    // largest row length among the chunks it covers
    auto launch_tiled = [&](int t_rows, int n_blocks, const AttnTile * tiles) {
        AttnTiledArgs ta{};
        ta.q16 = s->q16; ta.kc = kc; ta.vc = vc; ta.n_past = d_npast; ta.E = E; ta.H = H; ta.N = N; ta.texp = s->texp; ta.out = s->att;
        if (preq) { ta.aq_out = s->aq_att; ta.da_out = s->da_att; ta.out_nbq = s->nbqE; ta.out_dscale = dsc; ta.out_soff = s->soffE; }
        ta.kq_scale = kq_scale; ta.t_rows = t_rows; ta.t_pad = (t_rows + 31) & ~31;
        ta.tiles = tiles; ta.sess_stride = s->sess_stride;
        const size_t tsm = (size_t) ta.t_rows * kAttnRow + (size_t) kAttnQB * ta.t_pad * 6 + 4 * 8 * 128 * 4 + kAttnQB * 256 + 64;
        if (int e = smem_attr<k_attn128_tiled>(s, kSmemLimit)) return e;
        return launch(s, k_attn128_tiled, dim3(H, n_blocks, 1), dim3(512, 1, 1), tsm, ta);
    };
    // columns [c0, c0 + cnt) that are each an independent N = 1 step: the fused (RoPE + append) kernel, one cluster row per column
    auto launch_fused_cols = [&](int c0, int cnt) {
        for (int n0 = 0; n0 < cnt; n0 += kChunk) {
            aa.n0 = c0 + n0;
            if (int e = launch(s, k_attn128<true>, dim3(4 * H, std::min(cnt - n0, kChunk), 1), dim3(256, 1, 1), am.staged, aa)) return e;
        }
        return 0;
    };
    if (s->steps) {
        // decode rows: every row's K / V is appended first, then each row attends with T = its position + 1, the arithmetic
        // of its own single-token step.  Not the fused kernel: its columns would race on each other's K / V rows; not the
        // query-tiled one: it takes one T per chunk.
        s->cur_class = 1;
        RopeArgs ra{s->qkv, E, H, D, N, d_npast, s->cs, s->q16, kc, vc, s->cols, s->sess_stride};
        if ((rc = launch(s, k_rope_append, dim3((E / 2 + 255) / 256, N, 1), dim3(256, 1, 1), 0, ra))) return rc;
        s->cur_class = 2;
        aa.col_T = s->col_T;
        for (int n0 = 0; n0 < N; n0 += kChunk) {
            aa.n0 = n0;
            if ((rc = launch(s, k_attn128<false>, dim3(4 * H, std::min(N - n0, kChunk), 1), dim3(256, 1, 1), am.plain, aa))) return rc;
        }
        return 0;
    }
    if (s->cols && !s->col_T) {
        // batched step: every column is a single-token step
        s->cur_class = 2;
        return launch_fused_cols(0, N);
    }
    if (s->cols) {
        // Mixed pass.  A prompt segment's column j attends to the K / V rows its columns < j append in this layer, so the
        // fused kernel only serves the single-token segments (runs of adjacent ones share a launch).  The prompt segments are
        // appended first, then attended with T = the end of their segment: those within the staged window by one
        // query-tiled launch over the pass's tile table, the longer ones by the per-query cluster kernel.  All kernels are
        // on one stream, so every append is complete before an attention kernel reads the cache.
        const std::vector<b200_slice::Seg> & sg = s->segs;
        s->cur_class = 2;
        for (size_t k = 0; k < sg.size();) {
            size_t e = k;
            while (e < sg.size() && sg[e].count == 1) e++;
            if (e > k && (rc = launch_fused_cols(sg[k].col, sg[e - 1].col + 1 - sg[k].col))) return rc;
            k = e + 1;
        }
        s->cur_class = 1;
        for (const b200_slice::Seg & g : sg) {
            if (g.count == 1) continue;
            RopeArgs ra{s->qkv + (size_t) g.col * 3 * E, E, H, D, g.count, d_npast, s->cs, s->q16 + (size_t) g.col * E, kc, vc,
                        s->cols + g.col, s->sess_stride};
            if ((rc = launch(s, k_rope_append, dim3((E / 2 + 255) / 256, g.count, 1), dim3(256, 1, 1), 0, ra))) return rc;
        }
        s->cur_class = 2;
        if (s->n_tiles && (rc = launch_tiled(s->tile_rows, s->n_tiles, s->d_tiles))) return rc;
        aa.col_T = s->col_T;
        for (const b200_slice::Seg & g : sg) {
            if (g.count == 1 || seg_tiled(s, g)) continue;
            for (int n0 = 0; n0 < g.count; n0 += kChunk) {
                aa.n0 = g.col + n0;
                if ((rc = launch(s, k_attn128<false>, dim3(4 * H, std::min(g.count - n0, kChunk), 1), dim3(256, 1, 1), am.plain, aa))) return rc;
            }
        }
        return 0;
    }
    if (N == 1) {
        s->cur_class = 2;
        aa.n0 = 0;
        if (s->trace && s->trace_next < 512) { aa.trace = s->trace + (size_t) s->trace_next * 1024 * 8; s->trace_next++; s->trace_cls.push_back(2); s->trace_ctas.push_back(4 * H); }
        aa.lut_smem = s->attn_lut_smem;
        return launch(s, k_attn128<true>, dim3(4 * H, 1, 1), dim3(256, 1, 1), aa.lut_smem ? am.lut : am.staged, aa);
    }
    s->cur_class = 1;
    RopeArgs ra{s->qkv, E, H, D, N, d_npast, s->cs, s->q16, kc, vc, nullptr, 0};
    if ((rc = launch(s, k_rope_append, dim3((E / 2 + 255) / 256, N, 1), dim3(256, 1, 1), 0, ra))) return rc;
    s->cur_class = 2;
    if (s->use_tiled_attn && s->past[s->cur] + N <= kAttnTMax)
        // prompt chunk whose whole context fits the staged window: query-tiled kernel, K / V read once per 16 queries
        return launch_tiled(s->past[s->cur] + N, (N + kAttnQB - 1) / kAttnQB, nullptr);
    for (int n0 = 0; n0 < N; n0 += kChunk) {
        aa.n0 = n0;
        const int cnt = N - n0 < kChunk ? N - n0 : kChunk;
        if ((rc = launch(s, k_attn128<false>, dim3(4 * H, cnt, 1), dim3(256, 1, 1), am.plain, aa))) return rc;
    }
    return 0;
}

// ---------------------------------------------------------------- one layer per weight family
// Each enqueues layer il for N tokens: qkv -> attention -> wo -> w1|w3 -> w2, reading `cur` and writing `nxt`.
// Profile classes (cur_class): qkv 0, RoPE 1, attention 2, wo 3, w1|w3 4, w2 5; an input quantiser takes the class of
// the matmul it feeds.

// F16 weights: f32 activations, RMSNorm fused into the qkv and w1|w3 prologues
static int layer_f16(b200_slice * s, int il, int N, const float * cur, float * nxt) {
    const int E = s->E, FF = s->FF;
    const LayerW & Lw = s->layers[il];
    int rc;
    GemvF16Args q{}; q.K = E; q.x = cur; q.ldx = E; q.norm_w = Lw.attn_norm; q.N = N; q.tsilu = s->tsilu;
    q.rows = 3 * E; q.ldy = 3 * E;       // wq | wk | wv are packed back to back: one launch, one RMSNorm prologue
    q.W = Lw.f_q; q.y = s->qkv;
    if ((rc = launch_f16<PRO_NORM, EPI_STORE>(s, q))) return rc;
    if ((rc = attention(s, il, N, false))) return rc;
    s->cur_class = 3;
    GemvF16Args o{}; o.K = E; o.x = s->att; o.ldx = E; o.N = N; o.tsilu = s->tsilu;
    o.rows = E; o.W = Lw.f_o; o.resid = cur; o.ldr = E; o.y = s->ffin; o.ldy = E;
    if ((rc = launch_f16<PRO_PLAIN, EPI_RESID>(s, o))) return rc;
    s->cur_class = 4;
    GemvF16Args g{}; g.K = E; g.x = s->ffin; g.ldx = E; g.norm_w = Lw.ffn_norm; g.N = N; g.tsilu = s->tsilu;
    g.rows = FF; g.W = Lw.f_1; g.W2 = Lw.f_3; g.y = s->gate; g.ldy = FF;
    if ((rc = launch_f16<PRO_NORM, EPI_GATE>(s, g))) return rc;
    s->cur_class = 5;
    GemvF16Args w{}; w.K = FF; w.x = s->gate; w.ldx = FF; w.N = N; w.tsilu = s->tsilu;
    w.rows = E; w.W = Lw.f_2; w.resid = s->ffin; w.ldr = E; w.y = nxt; w.ldy = E;
    return launch_f16<PRO_PLAIN, EPI_RESID>(s, w);
}

// Block-quantised weights (Q4_0, Q4_1, Q5_0, Q5_1, Q8_0), bit-exact: every matmul input is quantised like the
// reference's, and where it can be, by the kernel that produces it (attention, the w1|w3 gate, the NQ epilogues)
static int layer_exact(b200_slice * s, int il, int N, const float * cur, float * nxt) {
    const int E = s->E, FF = s->FF;
    const LayerW & Lw = s->layers[il];
    // grid-barrier norm+quant epilogue: decode only (every CTA of wo / w2 must be co-resident: 1 tile per CTA)
    const bool nq = s->use_nq && N == 1 && !s->cols && Lw.wo.n_tiles <= 256 && Lw.wo.n_tiles <= s->n_sm * 2;
    const float dsc = wt_act_scale(s->wtype);
    int rc;
    GemvArgs q{}; q.W = Lw.qkv; q.x = cur; q.ldx = E; q.norm_w = Lw.attn_norm; q.y = s->qkv; q.ldy = 3 * E;
    q.N = N; q.out_rows = 3 * E; q.tsilu = s->tsilu; q.aq_in = s->aq_x; q.da_in = s->da_x; q.in_soff = s->soffE;
    // a multi-token call normalises + quantises every row ONCE instead of once per 32-row tile (k_norm_quant); with nq
    // the layers after the first get their input already normalised + quantised by the previous w2's last CTA
    if (N > 1 && (rc = launch_norm_quant(s, cur, E, Lw.attn_norm, N))) return rc;
    if ((rc = N > 1 || (il > 0 && nq) ? launch_gemv<1, PRO_PREQ, EPI_STORE>(s, q) : launch_gemv<1, PRO_NORM, EPI_STORE>(s, q))) return rc;
    if ((rc = attention(s, il, N, true))) return rc;
    s->cur_class = 3;
    GemvArgs o{}; o.W = Lw.wo; o.x = s->att; o.ldx = E; o.resid = cur; o.ldr = E; o.y = s->ffin; o.ldy = E;
    o.N = N; o.out_rows = E; o.tsilu = s->tsilu; o.aq_in = s->aq_att; o.da_in = s->da_att; o.in_soff = s->soffE; o.out_soff = s->soffE;
    o.nq_norm_w = Lw.ffn_norm; o.nq_counter = s->nq_counter; o.nq_partial = s->nq_partial; o.aq_out = s->aq_x; o.da_out = s->da_x; o.out_nbq = s->nbqE; o.out_dscale = dsc;
    if (s->D == 128) rc = nq ? launch_gemv<1, PRO_PREQ, EPI_RESID_NQ>(s, o) : launch_gemv<1, PRO_PREQ, EPI_RESID>(s, o);    // quantised by the attention
    else             rc = nq ? launch_gemv<1, PRO_PLAIN, EPI_RESID_NQ>(s, o) : launch_gemv<1, PRO_PLAIN, EPI_RESID>(s, o);
    if (rc) return rc;
    s->cur_class = 4;
    GemvArgs g{}; g.W = Lw.w13; g.x = s->ffin; g.ldx = E; g.norm_w = Lw.ffn_norm; g.y = s->gate; g.ldy = FF;
    g.N = N; g.out_rows = FF; g.tsilu = s->tsilu; g.aq_in = s->aq_x; g.da_in = s->da_x; g.in_soff = s->soffE; g.out_soff = s->soffF;
    g.aq_out = s->aq_gate; g.da_out = s->da_gate; g.out_nbq = s->nbqF; g.out_dscale = dsc;
    if (N > 1 && (rc = launch_norm_quant(s, s->ffin, E, Lw.ffn_norm, N))) return rc;
    if ((rc = N > 1 || nq ? launch_gemv<2, PRO_PREQ, EPI_GATEQ>(s, g) : launch_gemv<2, PRO_NORM, EPI_GATEQ>(s, g))) return rc;
    s->cur_class = 5;
    GemvArgs w{}; w.W = Lw.w2; w.resid = s->ffin; w.ldr = E; w.y = nxt; w.ldy = E;
    w.N = N; w.out_rows = E; w.tsilu = s->tsilu; w.aq_in = s->aq_gate; w.da_in = s->da_gate; w.in_soff = s->soffF; w.out_soff = s->soffE;
    if (il + 1 < s->L && nq) {
        w.nq_norm_w = s->layers[il + 1].attn_norm; w.nq_counter = s->nq_counter; w.nq_partial = s->nq_partial; w.aq_out = s->aq_x; w.da_out = s->da_x;
        w.out_nbq = s->nbqE; w.out_dscale = dsc;
        return launch_gemv<1, PRO_PREQ, EPI_RESID_NQ>(s, w);
    }
    if (s->fold_send && il == s->L - 1) return launch_w2_send<false>(s, w);
    return launch_gemv<1, PRO_PREQ, EPI_RESID>(s, w);
}

// Fast mode (Q4_0 / Q8_0 prompt chunks): each matmul's input goes through k_prep_q8_f16, the matmul through k_gemm_tc2
static int layer_fast(b200_slice * s, int il, int N, const float * cur, float * nxt) {
    const int E = s->E, FF = s->FF;
    const LayerW & Lw = s->layers[il];
    int rc;
    if ((rc = launch_prep<true>(s, cur, E, Lw.attn_norm, E, N))) return rc;
    if ((rc = launch_fast_gemm<FG_STORE>(s, Lw.qkv, nullptr, 0, s->qkv, 3 * E, N, 3 * E))) return rc;
    if ((rc = attention(s, il, N, true))) return rc;         // the quantised copy is written as in exact mode; wo reads s->att
    s->cur_class = 3;
    if ((rc = launch_prep<false>(s, s->att, E, nullptr, E, N))) return rc;
    if ((rc = launch_fast_gemm<FG_RESID>(s, Lw.wo, cur, E, s->ffin, E, N, E))) return rc;
    s->cur_class = 4;
    if ((rc = launch_prep<true>(s, s->ffin, E, Lw.ffn_norm, E, N))) return rc;
    if ((rc = launch_fast_gemm<FG_GATE>(s, Lw.w13, nullptr, 0, s->gate, FF, N, FF))) return rc;
    s->cur_class = 5;
    if ((rc = launch_prep<false>(s, s->gate, FF, nullptr, FF, N))) return rc;
    return launch_fast_gemm<FG_RESID>(s, Lw.w2, s->ffin, E, nxt, E, N, E);
}

// k-quant weights (Q4_K / Q6_K in any mix, kquant.cuh): every matmul input is quantised to Q8_K by quant_kq
static int layer_kquant(b200_slice * s, int il, int N, const float * cur, float * nxt) {
    const int E = s->E, FF = s->FF;
    const LayerW & Lw = s->layers[il];
    int rc;
    GemvArgs q{}; q.W = Lw.qkv; q.x = cur; q.ldx = E; q.norm_w = Lw.attn_norm; q.y = s->qkv; q.ldy = 3 * E;
    q.N = N; q.out_rows = Lw.qkv.rows; q.tsilu = s->tsilu;
    if ((rc = quant_kq(s, q, true)) || (rc = launch_gemv_kq<1, PRO_PREQ, EPI_STORE>(s, q))) return rc;
    for (int i = 0; i < 2 && Lw.qkv_more[i].data; i++) {       // wq | wk and wv of different types: same input and rows, exact
        q.W = Lw.qkv_more[i]; q.y = s->qkv + Lw.qkv_row[i]; q.out_rows = Lw.qkv_more[i].rows;
        if ((rc = launch_gemv_kq<1, PRO_PREQ, EPI_STORE>(s, q))) return rc;
    }
    if ((rc = attention(s, il, N, false))) return rc;        // wo quantises the f32 s->att itself
    s->cur_class = 3;
    GemvArgs o{}; o.W = Lw.wo; o.x = s->att; o.ldx = E; o.resid = cur; o.ldr = E; o.y = s->ffin; o.ldy = E;
    o.N = N; o.out_rows = E; o.tsilu = s->tsilu;
    if ((rc = quant_kq(s, o, false)) || (rc = launch_gemv_kq<1, PRO_PREQ, EPI_RESID>(s, o))) return rc;
    s->cur_class = 4;
    GemvArgs g{}; g.W = Lw.w13; g.x = s->ffin; g.ldx = E; g.norm_w = Lw.ffn_norm; g.y = s->gate; g.ldy = FF;
    g.N = N; g.out_rows = FF; g.tsilu = s->tsilu;
    if ((rc = quant_kq(s, g, true)) || (rc = launch_gemv_kq<2, PRO_PREQ, EPI_GATE>(s, g))) return rc;
    s->cur_class = 5;
    GemvArgs w{}; w.W = Lw.w2; w.x = s->gate; w.ldx = FF; w.resid = s->ffin; w.ldr = E; w.y = nxt; w.ldy = E;
    w.N = N; w.out_rows = E; w.tsilu = s->tsilu;
    if ((rc = quant_kq(s, w, false))) return rc;
    if (s->fold_send && il == s->L - 1) return launch_w2_send<true>(s, w);
    return launch_gemv_kq<1, PRO_PREQ, EPI_RESID>(s, w);
}

// ---------------------------------------------------------------- one forward over the slice
// Enqueue every layer for N tokens at device-side position *d_npast (tensor_processor.cpp:537-766).
static int enqueue_layers(b200_slice * s, const float * in, int N, float * out) {
    const float * cur = in;
    int rc;
    for (int il = 0; il < s->L; il++) {
        const LayerW & Lw = s->layers[il];
        float * nxt = (il == s->L - 1) ? out : ((il & 1) ? s->xb : s->xa);
        // fast mode is for single-session prefill calls only: a single-token step, a batched step or a mixed pass (cols:
        // columns of several sessions) stays exact, so decode, batch_forward and mixed_forward keep the reference's bits
        // whatever min_tokens is.  The windowed perplexity's fast mode (fast_pass) is the one caller that asks for it in
        // mixed passes: it only needs each window's rows close to exact
        const bool fast = N > 1 && ((s->fast_prefill && !s->cols && N >= s->fast_min_tokens) || s->fast_pass) &&
                          (s->wtype == kWT_Q4_0 || s->wtype == kWT_Q8_0) &&
                          (Lw.qkv.n_tiles * Lw.qkv.TR) % 16 == 0 &&
                          (Lw.wo.n_tiles * Lw.wo.TR) % 16 == 0 && (Lw.w13.n_tiles * Lw.w13.TR) % 16 == 0;
        s->cur_class = 0;
        if (s->wtype == kWT_F16)        rc = layer_f16(s, il, N, cur, nxt);
        else if (wt_kquant(s->wtype))   rc = layer_kquant(s, il, N, cur, nxt);
        else if (fast)                  rc = layer_fast(s, il, N, cur, nxt);
        else                            rc = layer_exact(s, il, N, cur, nxt);
        if (rc) return rc;
        cur = nxt;
    }
    s->cur_class = 6;
    if (s->send_pending) {
        // pipeline hand-off: the activation leaves for the next slice's GPU right behind the last matmul
        s->send_pending = false;
        if ((rc = launch(s, k_peer_send, dim3(s->send_ctas, 1, 1), dim3(1024, 1, 1), 0, s->send_args))) return rc;
    }
    if (s->cols) return launch(s, k_advance_segs, dim3(1), dim3(32), 0, s->d_npast, s->d_segs, (int) s->segs.size());
    if (s->fold_send) return launch(s, k_advance_sent, dim3(1), dim3(32), 0, s->d_npast + s->cur, N, (MailboxHdr *) s->mb_block);
    return launch(s, k_advance, dim3(1), dim3(32), 0, s->d_npast + s->cur, N);
}

// kernel launches of one captured single-token step over the slice (k-quant slices: + one k_quant_q8k per matmul input,
// + one launch per extra qkv run)
static int step_launches(const b200_slice * s) {
    int n = (s->D == 128 ? 5 : 6) * s->L + 1;
    for (const LayerW & Lw : s->layers) n += (Lw.qkv_more[0].data ? 1 : 0) + (Lw.qkv_more[1].data ? 1 : 0);
    if (wt_kquant(s->wtype)) n += 4 * s->L;
    return n;
}

// N = 1: replay a captured graph (host variant adds the H2D / D2H copies as graph nodes)
static int run_decode_graph(b200_slice * s, const float * in, float * out, bool host) {
    GraphKey key{in, out, (host ? 1 : 0) | (s->skip_attention ? 2 : 0) | (s->send_pending ? 4 : 0) | (s->cur << 3)};
    auto it = s->graphs.find(key);
    const int per_step = step_launches(s);
    if (it == s->graphs.end()) {
        const int64_t before = s->launches;
        cudaGraph_t g = nullptr;
        B200_CUDA(cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeThreadLocal));
        int rc = 0;
        if (host) {
            cudaMemcpyAsync(s->d_in, s->h_in, (size_t) s->E * 4, cudaMemcpyHostToDevice, s->stream);
            rc = enqueue_layers(s, s->d_in, 1, s->d_out);
            cudaMemcpyAsync(s->h_out, s->d_out, (size_t) s->E * 4, cudaMemcpyDeviceToHost, s->stream);
        } else {
            rc = enqueue_layers(s, in, 1, out);
        }
        cudaError_t e = cudaStreamEndCapture(s->stream, &g);
        s->launches = before;
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        if (e != cudaSuccess) return fail(B200_ECUDA, "graph capture failed: %s", cudaGetErrorString(e));
        cudaGraphExec_t ge = nullptr;
        e = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return fail(B200_ECUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
        if (s->graphs.size() >= 64)      // one graph per (buffers, session): enough for a node serving dozens of sessions
            { for (auto & kv : s->graphs) cudaGraphExecDestroy(kv.second); s->graphs.clear(); }
        it = s->graphs.emplace(key, ge).first;
    }
    B200_CUDA(cudaGraphLaunch(it->second, s->stream));
    s->launches += per_step;
    return 0;
}

static int forward_locked(b200_slice * s, const float * in, int N, float * out, bool host, int session = 0) {
    if (N <= 0) return fail(B200_EINVAL, "n_tokens must be positive (got %d)", N);
    if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    if (s->past[session] + N > s->n_ctx)
        return fail(B200_ECONTEXT, "context overflow: n_past %d + n_tokens %d > n_ctx %d", s->past[session], N, s->n_ctx);
    B200_CUDA(cudaSetDevice(s->device));
    s->cur = session; s->cols = nullptr;
    B200_CUDA(cudaEventRecord(s->ev0, s->stream));
    int rc;
    if (host) {
        if (N == 1 && s->use_graph && !s->profiling) {
            memcpy(s->h_in, in, (size_t) s->E * 4);
            if ((rc = run_decode_graph(s, nullptr, nullptr, true))) return rc;
            B200_CUDA(cudaEventRecord(s->ev1, s->stream));
            // A decoded token is ~1 ms of GPU work.  A blocking synchronize adds the wake-up latency of the driver's
            // interrupt path to every token; polling from the start burns a core for the whole token.  So: sleep through
            // ~70 % of the smoothed token time, poll the rest, and block if the token takes unusually long.
            if (s->ema_token_ms > 0.2f)
                std::this_thread::sleep_for(std::chrono::microseconds((long)(700.f * s->ema_token_ms)));
            for (int spin = 0; spin < 100000; spin++) if (cudaEventQuery(s->ev1) != cudaErrorNotReady) break;
            B200_CUDA(cudaStreamSynchronize(s->stream));
            { float ms = 0.f; if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) == cudaSuccess && ms > 0.f)
                  s->ema_token_ms = s->ema_token_ms > 0.f ? 0.8f * s->ema_token_ms + 0.2f * ms : ms; }
            memcpy(out, s->h_out, (size_t) s->E * 4);
        } else {
            B200_CUDA(cudaMemcpyAsync(s->d_in, in, (size_t) N * s->E * 4, cudaMemcpyHostToDevice, s->stream));
            if ((rc = enqueue_layers(s, s->d_in, N, s->d_out))) return rc;
            B200_CUDA(cudaEventRecord(s->ev1, s->stream));
            B200_CUDA(cudaMemcpyAsync(out, s->d_out, (size_t) N * s->E * 4, cudaMemcpyDeviceToHost, s->stream));
            B200_CUDA(cudaStreamSynchronize(s->stream));
        }
    } else {
        if (N == 1 && s->use_graph && !s->profiling) { if ((rc = run_decode_graph(s, in, out, false))) return rc; }
        else if ((rc = enqueue_layers(s, in, N, out))) return rc;
        B200_CUDA(cudaEventRecord(s->ev1, s->stream));
    }
    s->timed = true;
    s->past[session] += N;
    return 0;
}

// ---------------------------------------------------------------- batched and mixed passes
// One pass over n_seq distinct sessions: sessions[k] runs counts[k] tokens (counts == nullptr: one each) at its own
// positions past .. past + counts[k] - 1, and its rows follow those of sessions[k - 1].  The weight matmuls see every row
// as one column (weights read once); RoPE, the KV append and attention run per column against that session's cache.  Each
// session's rows are arithmetically those of b200_session_forward on that session alone, so results are bit-identical.
// Checks the whole list before anything moves; *total is the number of rows.
static int check_pass(const b200_slice * s, const int * sessions, const int * counts, int n_seq, int * total) {
    if (n_seq <= 0 || n_seq > s->n_sessions || n_seq > s->n_ctx) return fail(B200_EINVAL, "pass over %d sessions on a slice with %d sessions", n_seq, s->n_sessions);
    std::vector<char> seen(s->n_sessions, 0);
    long long rows = 0;
    for (int b = 0; b < n_seq; b++) {
        const int k = sessions[b], c = counts ? counts[b] : 1;
        if (k < 0 || k >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", k, s->n_sessions);
        if (seen[k]) return fail(B200_EINVAL, "session %d listed twice in one pass", k);
        seen[k] = 1;
        if (c <= 0) return fail(B200_EINVAL, "session %d: token count %d must be positive", k, c);
        if (s->past[k] + c > s->n_ctx)
            return fail(B200_ECONTEXT, "context overflow: session %d n_past %d + %d > n_ctx %d", k, s->past[k], c, s->n_ctx);
        rows += c;
    }
    if (rows > s->n_ctx) return fail(B200_EINVAL, "%lld rows in one pass exceed n_ctx %d", rows, s->n_ctx);
    *total = (int) rows;
    return 0;
}

// Builds the pass's tables (see b200_slice::segs) and uploads them in one copy on the slice's stream; from here until
// end_pass, enqueue_layers runs the pass.  An all-single-token pass (a batched step) has no row lengths and no tiles.
static int begin_pass(b200_slice * s, const int * sessions, const int * counts, int n_seq, int N) {
    std::vector<int> & h = s->h_pass;
    h.assign((size_t) 2 * N + 2 * n_seq, 0);
    s->segs.resize(n_seq);
    bool multi = false;
    for (int k = 0, col = 0; k < n_seq; k++) {
        const int id = sessions[k], c = counts ? counts[k] : 1, past = s->past[id];
        s->segs[k] = {id, past, c, col};
        for (int j = 0; j < c; j++) { h[2 * (col + j)] = id; h[2 * (col + j) + 1] = past + j; }
        h[2 * N + 2 * k] = id; h[2 * N + 2 * k + 1] = c;
        col += c; multi |= c > 1;
    }
    s->n_tiles = 0; s->tile_rows = 0;
    if (multi) {
        for (const b200_slice::Seg & g : s->segs)
            for (int j = 0; j < g.count; j++) h.push_back(g.past + g.count);
        for (const b200_slice::Seg & g : s->segs) {
            if (!seg_tiled(s, g)) continue;
            s->tile_rows = std::max(s->tile_rows, g.past + g.count);
            for (int q0 = 0; q0 < g.count; q0 += kAttnQB) { h.insert(h.end(), {g.session, g.past, g.count, q0, g.col + q0}); s->n_tiles++; }
        }
    }
    // pageable source: the driver stages it before returning
    B200_CUDA(cudaMemcpyAsync(s->d_pass, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, s->stream));
    s->cur = 0;
    s->cols = (const int2 *) s->d_pass;
    s->d_segs = (const int2 *)(s->d_pass + 2 * N);
    s->col_T = multi ? s->d_pass + 2 * N + 2 * n_seq : nullptr;
    s->d_tiles = s->n_tiles ? (const AttnTile *)(s->d_pass + 3 * N + 2 * n_seq) : nullptr;
    return 0;
}

static void end_pass(b200_slice * s) {
    s->cols = nullptr; s->col_T = nullptr; s->d_segs = nullptr; s->d_tiles = nullptr; s->n_tiles = 0; s->steps = false;
}

// Decode rows: N single-token steps of `session` in one pass, at the positions its DEVICE counter holds (k_steps_table), so
// the pass can follow device-side position updates without the host knowing them.  From here until end_pass,
// enqueue_layers runs the pass; its k_advance_segs moves the session N positions.  Fast prefill never applies (cols mode).
static int begin_steps(b200_slice * s, int session, int N) {
    if (int rc = launch(s, k_steps_table, dim3(1), dim3(256), 0, (const int *) s->d_npast, session, N, s->n_ctx, s->d_pass)) return rc;
    s->segs.assign(1, b200_slice::Seg{session, 0, N, 0});
    s->n_tiles = 0; s->tile_rows = 0; s->cur = 0; s->steps = true;
    s->cols = (const int2 *) s->d_pass;
    s->d_segs = (const int2 *)(s->d_pass + 2 * N);
    s->col_T = s->d_pass + 2 * N + 2;
    return 0;
}

// b200_session_forward_steps: decode rows with the host checks of b200_session_forward
static int steps_locked(b200_slice * s, int session, const float * in, int N, float * out, bool host) {
    if (N <= 0) return fail(B200_EINVAL, "n_tokens must be positive (got %d)", N);
    if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    if (s->past[session] + N > s->n_ctx)
        return fail(B200_ECONTEXT, "context overflow: n_past %d + n_tokens %d > n_ctx %d", s->past[session], N, s->n_ctx);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaEventRecord(s->ev0, s->stream));
    int rc;
    if ((rc = begin_steps(s, session, N))) { end_pass(s); return rc; }
    if (host) B200_CUDA(cudaMemcpyAsync(s->d_in, in, (size_t) N * s->E * 4, cudaMemcpyHostToDevice, s->stream));
    rc = enqueue_layers(s, host ? s->d_in : in, N, host ? s->d_out : out);
    end_pass(s);
    if (rc) return rc;
    B200_CUDA(cudaEventRecord(s->ev1, s->stream));
    if (host) {
        B200_CUDA(cudaMemcpyAsync(out, s->d_out, (size_t) N * s->E * 4, cudaMemcpyDeviceToHost, s->stream));
        B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    s->timed = true;
    s->past[session] += N;
    return 0;
}

static void advance_pass(b200_slice * s, const int * sessions, const int * counts, int n_seq) {
    for (int k = 0; k < n_seq; k++) s->past[sessions[k]] += counts ? counts[k] : 1;
}

// rows of the pass table: columns (session, position) and row lengths, segments, tiles
static size_t pass_table_ints(int n_ctx, int n_sessions) {
    return (size_t) 3 * n_ctx + 2 * (size_t) n_sessions + 5 * ((size_t) n_ctx / kAttnQB + n_sessions);
}

static int pass_locked(b200_slice * s, const int * sessions, const int * counts, int n_seq, const float * in, float * out, bool host) {
    int N = 0, rc;
    if ((rc = check_pass(s, sessions, counts, n_seq, &N))) return rc;
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaEventRecord(s->ev0, s->stream));
    if ((rc = begin_pass(s, sessions, counts, n_seq, N))) return rc;
    if (host) {
        B200_CUDA(cudaMemcpyAsync(s->d_in, in, (size_t) N * s->E * 4, cudaMemcpyHostToDevice, s->stream));
        rc = enqueue_layers(s, s->d_in, N, s->d_out);
        end_pass(s);
        if (rc) return rc;
        B200_CUDA(cudaEventRecord(s->ev1, s->stream));
        B200_CUDA(cudaMemcpyAsync(out, s->d_out, (size_t) N * s->E * 4, cudaMemcpyDeviceToHost, s->stream));
        B200_CUDA(cudaStreamSynchronize(s->stream));
    } else {
        rc = enqueue_layers(s, in, N, out);
        end_pass(s);
        if (rc) return rc;
        B200_CUDA(cudaEventRecord(s->ev1, s->stream));
    }
    s->timed = true;
    advance_pass(s, sessions, counts, n_seq);
    return 0;
}

// Element j of one 32-weight block of a block-quantised type, as ggml's dequantize_row_* computes it (ggml.c:1523-1633,
// built without contraction): q * d, and for Q4_1 / Q5_1 then + m (two roundings).
__device__ __forceinline__ float deq32(const uint8_t * blk, int type, int j) {
    const float d = h2f(*(const uint16_t *) blk);
    if (type == kWT_Q8_0) return fmul((float)((const int8_t *)(blk + 2))[j], d);
    if (type == kWT_Q4_0 || type == kWT_Q4_1) {
        const int q = blk[(type == kWT_Q4_1 ? 4 : 2) + (j & 15)], x = j < 16 ? (q & 0x0F) : (q >> 4);
        return type == kWT_Q4_1 ? fadd(fmul((float) x, d), h2f(*(const uint16_t *)(blk + 2))) : fmul((float)(x - 8), d);
    }
    const bool q51 = type == kWT_Q5_1;                    // Q5_0 / Q5_1
    const uint8_t * qh = blk + (q51 ? 4 : 2);
    const int q = qh[4 + (j & 15)];
    const int x = (j < 16 ? (q & 0x0F) : (q >> 4)) | (((qh[j >> 3] >> (j & 7)) & 1) << 4);
    return q51 ? fadd(fmul((float) x, d), h2f(*(const uint16_t *)(blk + 2))) : fmul((float)(x - 16), d);
}

// ---------------------------------------------------------------- LoRA merge (b200_slice_load_lora)
// llama_apply_lora_from_file_internal (llama.cpp:3054-3100) per matrix W [rows][K] with loraA (ne [r, K]) and loraB
// (ne [r, rows]):  BA = ggml_mul_mat(loraA, loraB), BA *= s when s = alpha / r != 1, then W += BA (or W = base + BA).
// One CTA takes one 32-column block of W and kLoraRows rows; a warp takes one row at a time, lane l column l, so the
// warp holds one whole quantisation block and requantises it with shuffles.
constexpr int kLoraRows = 64, kLoraWarps = 8;

struct LoraMergeArgs {
    const uint8_t * in;    // W's blocks / F16 values, or the base tensor (F16 / F32) when btype >= 0
    uint8_t * out;         // W-type output (== in when there is no base: each warp reads its block before it writes it)
    const float * A, * B;  // [K][r], [rows][r]
    int r, K, rows, wtype, btype;
    float scale; int scaled;
};

// ggml_vec_dot_f32 (ggml.c:2286) in the AVX2 + FMA build: lane m of accumulator j sums x[i]*y[i] for i = 32c + 8j + m
// with one FMA per element, GGML_F32x8_REDUCE (ggml.c:1895) folds the 32 partial sums in a fixed tree, and the last
// r % 32 products are added one by one (multiply, then add).
__device__ __forceinline__ float lora_dot(const float * As, const float * Bs, int r, int lane) {
    const int np = r & ~31;
    float sum = 0.f;
    if (np) {
        auto P = [&](int i) { float acc = 0.f; for (int c = 0; c < np; c += 32) acc = __fmaf_rn(As[(c + i) * 32 + lane], Bs[c + i], acc); return acc; };
        auto V = [&](int m) { return fadd(fadd(P(m), P(16 + m)), fadd(P(8 + m), P(24 + m))); };   // (x0 + x2) + (x1 + x3)
        sum = fadd(fadd(fadd(V(0), V(4)), fadd(V(1), V(5))), fadd(fadd(V(2), V(6)), fadd(V(3), V(7))));
    }
    for (int i = np; i < r; i++) sum = fadd(sum, fmul(As[i * 32 + lane], Bs[i]));
    return sum;
}

// The warp's first lane (in lane order) whose v wins under `better`; ties keep the lower lane, as a forward scan with a
// strict comparison does.
template <typename F> __device__ __forceinline__ float warp_pick(float v, F better) {
    int idx = threadIdx.x & 31;
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (better(ov, v) || (!better(v, ov) && oi < idx)) { v = ov; idx = oi; }
    }
    return v;
}

// Lane l holds element l of a block; writes it as one `type` block (ggml.c quantize_row_*_reference for the 4- and
// 5-bit types, the AVX2 quantize_row_q8_0 for Q8_0: that is type_traits[type].from_float, ggml.c:1655-1690).
__device__ void quant32(float x, int type, uint8_t * blk) {
    const int lane = threadIdx.x & 31;
    if (type == kWT_Q8_0) {                                  // ggml.c:1180-1240: id = 127 / amax, round half to even
        float amax = fabsf(x);
        for (int o = 16; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float d = __fdiv_rn(amax, 127.f), id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
        const int q = __float2int_rn(fmul(x, id));
        if (lane == 0) *(uint16_t *) blk = __half_as_ushort(__float2half_rn(d));
        blk[2 + lane] = (uint8_t)(int8_t) q;
        return;
    }
    int xi;
    float d, m = 0.f;
    if (type == kWT_Q4_0 || type == kWT_Q5_0) {              // max = the first v of largest |v| (0 when every v is 0)
        const float half = type == kWT_Q4_0 ? 8.f : 16.f;
        float mx = warp_pick(x, [](float a, float b) { return fabsf(a) > fabsf(b); });
        if (fabsf(mx) == 0.f) mx = 0.f;
        d = __fdiv_rn(mx, -half);
        const float id = d != 0.f ? __fdiv_rn(1.f, d) : 0.f;
        xi = min(type == kWT_Q4_0 ? 15 : 31, __float2int_rz(fadd(fmul(x, id), half + 0.5f)));
    } else {                                                 // Q4_1 / Q5_1: the first minimum and maximum
        const bool q41 = type == kWT_Q4_1;
        m = warp_pick(x, [](float a, float b) { return a < b; });
        const float mx = warp_pick(x, [](float a, float b) { return a > b; });
        d = __fdiv_rn(fsub(mx, m), q41 ? 15.f : 31.f);
        const float id = d != 0.f ? __fdiv_rn(1.f, d) : 0.f;
        xi = __float2int_rz(fadd(fmul(fsub(x, m), id), 0.5f));
        xi = q41 ? min(15, xi) : (xi & 0xFF);
    }
    const int hi = __shfl_down_sync(0xffffffffu, xi, 16);
    const unsigned qh = __ballot_sync(0xffffffffu, (xi & 0x10) != 0);
    const bool has_m = type == kWT_Q4_1 || type == kWT_Q5_1, five = type == kWT_Q5_0 || type == kWT_Q5_1;
    uint8_t * qs = blk + 2 + (has_m ? 2 : 0) + (five ? 4 : 0);
    if (lane < 16) qs[lane] = (uint8_t)((xi & 0x0F) | ((hi & 0x0F) << 4));
    if (lane == 0) {
        *(uint16_t *) blk = __half_as_ushort(__float2half_rn(d));
        if (has_m) *(uint16_t *)(blk + 2) = __half_as_ushort(__float2half_rn(m));
    }
    if (five && lane < 4) blk[2 + (has_m ? 2 : 0) + lane] = (uint8_t)(qh >> (8 * lane));
}

__global__ void __launch_bounds__(kLoraWarps * 32) k_lora_merge(LoraMergeArgs a) {
    extern __shared__ float lsm[];
    float * As = lsm;                                        // [r][32]: the block's 32 columns of loraA, k-major
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cb = blockIdx.x, c = cb * 32 + lane;
    float * Bs = lsm + (size_t) a.r * 32 + (size_t) warp * a.r;
    for (int i = threadIdx.x; i < 32 * a.r; i += blockDim.x) {
        const int l = i / a.r, k = i - l * a.r;
        As[k * 32 + l] = a.A[(size_t)(cb * 32 + l) * a.r + k];
    }
    __syncthreads();
    const int nb = a.K / 32, row_end = min(a.rows, (int)(blockIdx.y + 1) * kLoraRows);
    for (int j = blockIdx.y * kLoraRows + warp; j < row_end; j += kLoraWarps) {
        for (int k = lane; k < a.r; k += 32) Bs[k] = a.B[(size_t) j * a.r + k];
        __syncwarp();
        float ba = lora_dot(As, Bs, a.r, lane);
        if (a.scaled) ba = fmul(ba, a.scale);                // ggml_vec_scale_f32
        const size_t e = (size_t) j * a.K + c;
        float x;
        if (a.btype == kWT_F16) {                            // ggml_add of an F16 base gives an F16 tensor
            const uint16_t h = __half_as_ushort(__float2half_rn(fadd(h2f(((const uint16_t *) a.in)[e]), ba)));
            if (a.wtype == kWT_F16) { ((uint16_t *) a.out)[e] = h; __syncwarp(); continue; }
            x = h2f(h);
        } else if (a.btype == 0) {                           // F32 base
            x = fadd(((const float *) a.in)[e], ba);
        } else if (a.wtype == kWT_F16) {                     // ggml_compute_forward_add_f16_f32 (ggml.c:8375)
            x = fadd(h2f(((const uint16_t *) a.in)[e]), ba);
        } else {                                             // ggml_compute_forward_add_q_f32 (ggml.c:8483)
            x = fadd(deq32(a.in + ((size_t) j * nb + cb) * wt_traits(a.wtype).block_bytes, a.wtype, lane), ba);
        }
        __syncwarp();                                        // every lane has read the block before it is overwritten
        if (a.wtype == kWT_F16) ((uint16_t *) a.out)[e] = __half_as_ushort(__float2half_rn(x));
        else quant32(x, a.wtype, a.out + ((size_t) j * nb + cb) * wt_traits(a.wtype).block_bytes);
        __syncwarp();
    }
}

static size_t lora_smem(int r) { return (size_t)(32 + kLoraWarps) * r * sizeof(float); }

// ---------------------------------------------------------------- loader
// file (mmap, page cache) --reader thread--> pinned staging ring --DMA--> device scratch ring --k_repack--> packed HBM.
// Three slots are in flight: while slot j is repacked on the GPU, slot j+1 is on the PCIe bus and the reader thread is
// faulting slot j+2 in from the page cache.  Nothing synchronises the stream per matrix; a slot is reused once the
// event recorded behind its repack kernel has completed (the reader thread waits for it).
struct LoadJob {
    const GgjtTensor * src[3] = {nullptr, nullptr, nullptr};
    int nsrc = 0;
    int kind = 0;                 // 0: block-quantised or k-quant matrix (k_repack, k_repack_kq), 1: F16 (k_repack_f16), 2: raw copy
    int mode = 0, G = 1;
    PackedW * out = nullptr;      // kind 0
    uint16_t ** outf = nullptr; uint16_t * into = nullptr;   // kind 1
    uint8_t * raw_dst = nullptr;  // kind 2
    // LoRA (b200_slice_load_lora): source i is merged on the device before the repack.  With a base file, base[i] (F16
    // or F32) is uploaded in its place and the merge writes source-type blocks into a region behind the uploaded ones.
    const struct LoraPair * lora[3] = {nullptr, nullptr, nullptr};
    const GgjtTensor * base[3] = {nullptr, nullptr, nullptr};
    const GgjtFile * base_file = nullptr;
    static size_t al(size_t n) { return (n + 255) & ~(size_t) 255; }
    const GgjtTensor & up(int i) const { return base[i] ? *base[i] : *src[i]; }
    size_t up_bytes() const { size_t n = 0; for (int i = 0; i < nsrc; i++) n += al(up(i).nbytes); return n; }
    size_t bytes() const { size_t n = up_bytes(); for (int i = 0; i < nsrc; i++) if (base[i]) n += al(src[i]->nbytes); return n; }
    // where source i's uploaded bytes, and its (merged) source-type bytes, sit in a slot
    uint8_t * up_at(uint8_t * slot, int i) const { size_t o = 0; for (int k = 0; k < i; k++) o += al(up(k).nbytes); return slot + o; }
    uint8_t * src_at(uint8_t * slot, int i) const {
        if (!base[i]) return up_at(slot, i);
        size_t o = up_bytes();
        for (int k = 0; k < i; k++) if (base[k]) o += al(src[k]->nbytes);
        return slot + o;
    }
};

// One adapted matrix: loraA [K][r] and loraB [rows][r] in device memory
struct LoraPair { const float * A = nullptr, * B = nullptr; int r = 0; };
struct LoraMerge { float scale = 1.f; int scaled = 0; };

struct LoadPipe {
    static constexpr int NB = 3;
    uint8_t * pinned[NB] = {nullptr, nullptr, nullptr};
    uint8_t * scratch[NB] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev[NB] = {nullptr, nullptr, nullptr};
    size_t slot_bytes = 0;
    ~LoadPipe() {
        for (int i = 0; i < NB; i++) {
            if (pinned[i]) cudaFreeHost(pinned[i]);
            if (scratch[i]) cudaFree(scratch[i]);
            if (ev[i]) cudaEventDestroy(ev[i]);
        }
    }
};

static int run_load_jobs(b200_slice * s, const GgjtFile & f, std::vector<LoadJob> & jobs, const LoraMerge & lm = LoraMerge()) {
    if (jobs.empty()) return 0;
    LoadPipe lp;
    for (const LoadJob & j : jobs) lp.slot_bytes = std::max(lp.slot_bytes, j.bytes());
    lp.slot_bytes += 4096;
    for (int i = 0; i < LoadPipe::NB; i++) {
        B200_CUDA(cudaMallocHost((void **) &lp.pinned[i], lp.slot_bytes));
        B200_CUDA(cudaMalloc((void **) &lp.scratch[i], lp.slot_bytes));
        B200_CUDA(cudaEventCreateWithFlags(&lp.ev[i], cudaEventDisableTiming));
    }
    posix_fadvise(f.fd, 0, 0, POSIX_FADV_SEQUENTIAL);       // a cold file: deep kernel read-ahead in front of the preads
    std::mutex mu; std::condition_variable cv;
    size_t filled = 0, consumed = 0; bool abort_flag = false;
    const int device = s->device;
    std::thread reader([&] {
        cudaSetDevice(device);
        for (size_t j = 0; j < jobs.size(); j++) {
            const int slot = (int)(j % LoadPipe::NB);
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return abort_flag || consumed + LoadPipe::NB > j; });
                if (abort_flag) return;
            }
            if (j >= LoadPipe::NB) cudaEventSynchronize(lp.ev[slot]);    // the slot's previous repack has read its scratch
            // pread straight into the pinned slot: page-cache copy without the per-4-KiB minor faults a private file
            // mapping costs; the job is cut in two so a second thread overlaps its copy
            struct Piece { uint8_t * dst; size_t off, n; const GgjtFile * file; };
            std::vector<Piece> pieces;
            size_t off = 0;
            for (int i = 0; i < jobs[j].nsrc; i++) {
                const GgjtTensor & t = jobs[j].up(i);
                const GgjtFile * tf = jobs[j].base[i] ? jobs[j].base_file : &f;
                const size_t half = (t.nbytes / 2) & ~(size_t) 4095;
                pieces.push_back({lp.pinned[slot] + off, t.offset, half, tf});
                pieces.push_back({lp.pinned[slot] + off + half, t.offset + half, t.nbytes - half, tf});
                off += (t.nbytes + 255) & ~(size_t) 255;
            }
            auto pull = [&](int first) {
                for (size_t k = first; k < pieces.size(); k += 2) {
                    size_t done = 0;
                    const GgjtFile & pf = *pieces[k].file;
                    while (done < pieces[k].n) {
                        const ssize_t got = pread(pf.fd, pieces[k].dst + done, pieces[k].n - done, (off_t)(pieces[k].off + done));
                        if (got <= 0) { memcpy(pieces[k].dst + done, pf.base + pieces[k].off + done, pieces[k].n - done); break; }
                        done += (size_t) got;
                    }
                }
            };
            std::thread helper(pull, 1);
            pull(0);
            helper.join();
            { std::lock_guard<std::mutex> lk(mu); filled = j + 1; }
            cv.notify_all();
        }
    });
    int rc = 0;
    for (size_t j = 0; j < jobs.size() && !rc; j++) {
        const int slot = (int)(j % LoadPipe::NB);
        LoadJob & job = jobs[j];
        { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return filled > j; }); }
        cudaError_t e = cudaMemcpyAsync(lp.scratch[slot], lp.pinned[slot], job.up_bytes(), cudaMemcpyHostToDevice, s->stream);
        if (e != cudaSuccess) { rc = fail(B200_ECUDA, "weight upload failed: %s", cudaGetErrorString(e)); break; }
        for (int i = 0; i < job.nsrc; i++) {
            if (!job.lora[i]) continue;
            const GgjtTensor & t = *job.src[i];
            LoraMergeArgs la{};
            la.in = job.up_at(lp.scratch[slot], i); la.out = job.src_at(lp.scratch[slot], i);
            la.A = job.lora[i]->A; la.B = job.lora[i]->B; la.r = job.lora[i]->r;
            la.K = (int) t.ne[0]; la.rows = (int) t.ne[1]; la.wtype = (int) t.type;
            la.btype = job.base[i] ? (int) job.base[i]->type : -1;
            la.scale = lm.scale; la.scaled = lm.scaled;
            k_lora_merge<<<dim3(la.K / 32, (la.rows + kLoraRows - 1) / kLoraRows), kLoraWarps * 32, lora_smem(la.r), s->stream>>>(la);
        }
        if (job.kind == 0) {
            const int wt = (int) job.src[0]->type;
            const bool kqt = wt_kquant(wt);             // k-quants: nb / nbq count 256-wide super-blocks
            const int K = (int) job.src[0]->ne[0], rows_per = (int) job.src[0]->ne[1];
            const int nb = kqt ? K / 256 : K / 32, TR = kWPC * job.G;
            const int nbq = kqt ? (nb + kKQS - 1) / kKQS * kKQS : ((nb + 3) / 4 + kQS - 1) / kQS * kQS;
            const int total_groups = (rows_per + 7) / 8 * job.nsrc;
            const int n_tiles = (total_groups + TR - 1) / TR;
            const long long tile_bytes = (long long) nbq * TR * (kqt ? kq_chunk_bytes(wt) : chunk_bytes(wt));
            uint8_t * dst = nullptr;
            if ((rc = dev_alloc(s, &dst, (size_t) n_tiles * tile_bytes))) break;
            RepackArgs ra{};
            for (int i = 0; i < job.nsrc; i++) ra.src[i] = job.src_at(lp.scratch[slot], i);
            ra.mode = job.mode; ra.wtype = wt; ra.rows_per_src = rows_per; ra.nb = nb; ra.nbq = nbq; ra.TR = TR; ra.n_tiles = n_tiles;
            ra.dst = dst;
            if (kqt) k_repack_kq<<<s->n_sm * 8, 256, 0, s->stream>>>(ra);
            else k_repack<<<s->n_sm * 8, 256, 0, s->stream>>>(ra);
            PackedW * out = job.out;
            out->data = dst; out->wtype = wt; out->rows = rows_per * job.nsrc; out->K = K; out->nb = nb; out->nbq = nbq; out->TR = TR;
            out->n_tiles = n_tiles; out->tile_bytes = tile_bytes;
        } else if (job.kind == 1) {
            const GgjtTensor & t = *job.src[0];
            const int K = (int) t.ne[0], rows = (int) t.ne[1];
            const int nchunk = K / 32, nc8 = (nchunk + 7) / 8;
            uint16_t * dst = job.into;
            if (!dst && (rc = dev_alloc(s, &dst, (size_t) rows * nc8 * 256 + 8))) break;
            k_repack_f16<<<s->n_sm * 8, 256, 0, s->stream>>>((const uint16_t *) job.src_at(lp.scratch[slot], 0), dst, dst /*no tail: K%32==0*/, rows, K);
            *job.outf = dst;
        } else {
            e = cudaMemcpyAsync(job.raw_dst, lp.scratch[slot], job.src[0]->nbytes, cudaMemcpyDeviceToDevice, s->stream);
            if (e != cudaSuccess) { rc = fail(B200_ECUDA, "weight copy failed: %s", cudaGetErrorString(e)); break; }
        }
        if ((e = cudaGetLastError()) != cudaSuccess) { rc = fail(B200_ECUDA, "repack launch failed: %s", cudaGetErrorString(e)); break; }
        cudaEventRecord(lp.ev[slot], s->stream);
        { std::lock_guard<std::mutex> lk(mu); consumed = j + 1; }
        cv.notify_all();
    }
    { std::lock_guard<std::mutex> lk(mu); abort_flag = rc != 0; consumed = jobs.size() + LoadPipe::NB; }
    cv.notify_all();
    reader.join();
    cudaError_t e = cudaStreamSynchronize(s->stream);
    if (!rc && e != cudaSuccess) rc = fail(B200_ECUDA, "weight repack failed: %s", cudaGetErrorString(e));
    return rc;
}

static int build_tables(b200_slice * s) {
    // fp16 lookup tables of ggml_init (ggml.c:4300-4312), built with the host libm like the reference does
    std::vector<uint16_t> texp(65536), tsilu(65536);
    for (int i = 0; i < 65536; i++) {
        const float f = __half2float(__ushort_as_half((unsigned short) i));
        texp[i]  = __half_as_ushort(__float2half_rn(expf(f)));
        tsilu[i] = __half_as_ushort(__float2half_rn(f / (1.0f + expf(-f))));
    }
    int rc;
    if ((rc = dev_alloc(s, &s->texp, 65536)) || (rc = dev_alloc(s, &s->tsilu, 65536))) return rc;
    B200_CUDA(cudaMemcpy(s->texp, texp.data(), 65536 * 2, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMemcpy(s->tsilu, tsilu.data(), 65536 * 2, cudaMemcpyHostToDevice));
    // RoPE cos/sin, theta iterated in f32 (ggml.c:12000, 12038-12044)
    const int half = s->D / 2;
    std::vector<float2> cs((size_t) s->n_ctx * half);
    const float theta_scale = powf(10000.0, -2.0f / s->D);
    for (int p = 0; p < s->n_ctx; p++) {
        float theta = (float) p;
        for (int j = 0; j < half; j++) {
            cs[(size_t) p * half + j] = make_float2(cosf(theta), sinf(theta));
            theta *= theta_scale;
        }
    }
    if ((rc = dev_alloc(s, &s->cs, cs.size()))) return rc;
    B200_CUDA(cudaMemcpy(s->cs, cs.data(), cs.size() * sizeof(float2), cudaMemcpyHostToDevice));
    return 0;
}

// ---------------------------------------------------------------- LoRA adapter plan
constexpr int kLoraMaxRank = 1024;      // loraA's 32 columns of one block stay in shared memory (160 KB at this rank)

// What an adapter contributes to one load: the parsed files, loraA / loraB of every adapted matrix in device memory
// (freed when the load ends), and the merge's scale.
struct LoraState {
    std::unique_ptr<GglaFile> ad;
    std::unique_ptr<GgjtFile> base;
    float * dev = nullptr;
    std::vector<LoraPair> pairs;
    LoraMerge merge;
    ~LoraState() { if (dev) cudaFree(dev); }
};

// layers.N.attention.w{q,k,v,o}.weight or layers.N.feed_forward.w{1,2,3}.weight: its layer N
static bool lora_target(const std::string & n, int * layer) {
    if (n.compare(0, 7, "layers.") != 0) return false;
    size_t q = 7;
    while (q < n.size() && isdigit((unsigned char) n[q])) q++;
    if (q == 7 || q - 7 > 6 || q >= n.size() || n[q] != '.') return false;
    const std::string rest = n.substr(q + 1);
    for (const char * m : {"attention.wq.weight", "attention.wk.weight", "attention.wv.weight", "attention.wo.weight",
                           "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight"})
        if (rest == m) { *layer = atoi(n.c_str() + 7); return true; }
    return false;
}

static std::string ne_str(const std::vector<uint32_t> & ne) {
    std::string r = "[";
    for (size_t i = 0; i < ne.size(); i++) r += (i ? ", " : "") + std::to_string(ne[i]);
    return r + "]";
}

// Checks the adapter (and base) against slice file f, uploads loraA / loraB of every matrix of the slice it adapts, and
// points the jobs' sources at them.  Nothing is repacked yet, so a refusal here leaves nothing behind but what the
// failed load frees anyway.
static int plan_lora(b200_slice * s, const GgjtFile & f, const char * lora_path, const char * base_path,
                     std::vector<LoadJob> & jobs, LoraState & st) {
    try { st.ad.reset(new GglaFile(lora_path)); }
    catch (const std::exception & e) { return fail(B200_EFILE, "error loading LoRA adapter: %s", e.what()); }
    if (base_path) {
        try { st.base.reset(new GgjtFile(base_path, false)); }
        catch (const std::exception & e) { return fail(B200_EFILE, "error loading LoRA base: %s", e.what()); }
    }
    const GglaFile & ad = *st.ad;
    struct Pair { const GgjtTensor * a = nullptr, * b = nullptr, * w = nullptr, * bw = nullptr; };
    std::map<std::string, Pair> by;                   // adapted matrices of this slice, by W's name
    for (const GgjtTensor & t : ad.tensors) {
        const size_t pos = t.name.rfind(".lora");
        const std::string kind = pos == std::string::npos ? "" : t.name.substr(pos + 5);
        if (kind != "A" && kind != "B")
            return fail(B200_EFILE, "adapter tensor '%s' is not a LoRA tensor (its name must end in .loraA or .loraB)", t.name.c_str());
        const std::string bn = t.name.substr(0, pos);
        int layer = -1;
        if (!lora_target(bn, &layer))
            return fail(B200_EFILE, "adapter tensor '%s': '%s' is not a layer matrix (layers.N.attention.wq/wk/wv/wo.weight, "
                                    "layers.N.feed_forward.w1/w2/w3.weight)", t.name.c_str(), bn.c_str());
        if (t.ne.size() != 2)
            return fail(B200_EFILE, "adapter tensor '%s' has %zu dimensions; LoRA tensors are 2-D", t.name.c_str(), t.ne.size());
        if (t.type != GT_F32)
            return fail(B200_EFILE, "adapter tensor '%s' is F16; LoRA tensors must be F32 (convert the checkpoint's loraA to float32)",
                        t.name.c_str());
        if (layer < s->first_layer || layer >= s->first_layer + s->L) continue;   // another slice's layer
        Pair & p = by[bn];
        const GgjtTensor *& slot = kind == "A" ? p.a : p.b;
        if (slot) return fail(B200_EFILE, "adapter tensor '%s' appears twice", t.name.c_str());
        slot = &t;
    }
    size_t floats = 0;
    int max_r = 0;
    for (auto & kv : by) {
        Pair & p = kv.second;
        const std::string & bn = kv.first;
        if (!p.a || !p.b)
            return fail(B200_EFILE, "adapter has %s.lora%s but no %s.lora%s for this slice's matrix (a lone A or B is refused)",
                        bn.c_str(), p.a ? "A" : "B", bn.c_str(), p.a ? "B" : "A");
        auto it = f.index.find(bn);
        if (it == f.index.end()) return fail(B200_EFILE, "adapter tensor '%s.loraA': the slice has no %s", bn.c_str(), bn.c_str());
        p.w = &f.tensors[it->second];
        if (wt_kquant((int) p.w->type))
            return fail(B200_EFILE, "adapter targets %s, a k-quant matrix (type %u): LoRA on Q4_K / Q6_K matrices is not supported",
                        bn.c_str(), p.w->type);
        const uint32_t r = p.a->ne[0];
        if (p.b->ne[0] != r)
            return fail(B200_EFILE, "adapter tensors %s.loraA (rank %u) and %s.loraB (rank %u) differ in rank", bn.c_str(), r,
                        bn.c_str(), p.b->ne[0]);
        if (p.a->ne[1] != p.w->ne[0] || p.b->ne[1] != p.w->ne[1])
            return fail(B200_EFILE, "adapter tensors %s.loraA %s / .loraB %s do not fit %s %s (want [r, %u] and [r, %u])", bn.c_str(),
                        ne_str(p.a->ne).c_str(), ne_str(p.b->ne).c_str(), bn.c_str(), ne_str(p.w->ne).c_str(), p.w->ne[0], p.w->ne[1]);
        if (r == 0 || r > (uint32_t) kLoraMaxRank)
            return fail(B200_EFILE, "adapter tensor %s.loraA has rank %u (supported: 1 .. %d)", bn.c_str(), r, kLoraMaxRank);
        if (st.base) {
            auto bt = st.base->index.find(bn);
            if (bt == st.base->index.end()) return fail(B200_EFILE, "LoRA base lacks tensor '%s'", bn.c_str());
            p.bw = &st.base->tensors[bt->second];
            if (p.bw->ne != p.w->ne)
                return fail(B200_EFILE, "LoRA base tensor '%s' has shape %s, the slice's has %s", bn.c_str(), ne_str(p.bw->ne).c_str(),
                            ne_str(p.w->ne).c_str());
            if (p.bw->type != GT_F16 && p.bw->type != GT_F32)
                return fail(B200_EFILE, "LoRA base tensor '%s' has type %u; a base must be F16 (1) or F32 (0)", bn.c_str(), p.bw->type);
        }
        floats += (p.a->nbytes + p.b->nbytes) / 4;
        max_r = std::max(max_r, (int) r);
    }
    if (by.empty()) return 0;                         // the adapter touches nothing here: a plain load
    B200_CUDA(cudaMalloc((void **) &st.dev, floats * 4));
    st.pairs.resize(by.size());
    std::map<std::string, const LoraPair *> pair_of;
    size_t off = 0, k = 0;
    for (auto & kv : by) {
        LoraPair & lp = st.pairs[k++];
        lp.r = (int) kv.second.a->ne[0];
        lp.A = st.dev + off;
        B200_CUDA(cudaMemcpy(st.dev + off, ad.data(*kv.second.a), kv.second.a->nbytes, cudaMemcpyHostToDevice));
        off += kv.second.a->nbytes / 4;
        lp.B = st.dev + off;
        B200_CUDA(cudaMemcpy(st.dev + off, ad.data(*kv.second.b), kv.second.b->nbytes, cudaMemcpyHostToDevice));
        off += kv.second.b->nbytes / 4;
        pair_of[kv.first] = &lp;
    }
    for (LoadJob & j : jobs)
        for (int i = 0; i < j.nsrc; i++) {
            auto it = pair_of.find(j.src[i]->name);
            if (it == pair_of.end()) continue;
            j.lora[i] = it->second;
            if (st.base) { j.base[i] = by[it->first].bw; j.base_file = st.base.get(); }
        }
    st.merge.scale = (float) ad.alpha / (float) ad.r;    // llama.cpp:2878
    st.merge.scaled = st.merge.scale != 1.0f;
    if (lora_smem(max_r) > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(k_lora_merge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) lora_smem(max_r)));
    return 0;
}

static int load_locked(b200_slice * s, const char * path, const char * lora_path = nullptr, const char * base_path = nullptr) {
    const bool ltrace = env_int("B200_LOAD_TRACE", 0) != 0;
    auto tnow = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_begin = tnow(); double t_last = t_begin;
    auto lap = [&](const char * what) { if (ltrace) { const double t = tnow(); fprintf(stderr, "[b200 load] %-28s %7.3f s\n", what, t - t_last); t_last = t; } };
    std::unique_ptr<GgjtFile> fp;
    try { fp.reset(new GgjtFile(path, false)); }
    catch (const std::exception & e) { return fail(B200_EFILE, "error loading model: %s", e.what()); }
    GgjtFile & f = *fp;
    lap("parse header + tensor index");
    if (f.n_layer == 0 || f.n_head == 0 || f.n_embd % f.n_head || f.n_embd % 32)
        return fail(B200_EFILE, "not a transformer slice file (n_layer=%u n_embd=%u n_head=%u)", f.n_layer, f.n_embd, f.n_head);
    s->E = (int) f.n_embd; s->H = (int) f.n_head; s->D = s->E / s->H; s->L = (int) f.n_layer; s->first_layer = (int) f.first_layer;
    s->FF = (int)(((2 * (4 * f.n_embd) / 3 + f.n_mult - 1) / f.n_mult) * f.n_mult);   // tensor_processor.cpp:1250
    if (s->D > 128 || (s->D & 1)) return fail(B200_EFILE, "head size %d unsupported (<=128, even)", s->D);
    // worst-case dynamic shared memory of the attention kernels at this n_ctx (the single-token kernel with the exp table
    // staged, or k_attention): reject the load instead of failing every forward later
    const AttnSmem am = attn_smem(s->n_ctx, s->D);
    const size_t attn_need = s->D == 128 ? am.lut : am.generic, attn_limit = s->D == 128 ? (size_t) 200 * 1024 : (size_t) kSmemLimit;
    if (attn_need > attn_limit)
        return fail(B200_EINVAL, "n_ctx %d needs %zu B of attention shared memory (limit %zu B): largest supported n_ctx for head size %d is %d",
                    s->n_ctx, attn_need, attn_limit, s->D, s->D == 128 ? (int)((attn_limit - 2 * 128 * kAttnRow - 32 * 64 - 64 - 65536 - 16) / 6) & ~31
                                                                       : (int)((attn_limit - (size_t) 4 * s->D * 32 - 64) / 6) & ~31);
    const uint32_t E = f.n_embd, FF = (uint32_t) s->FF;
    s->layers.resize(s->L);
    int rc;
    std::vector<LoadJob> jobs;
    std::vector<float> norms;                       // all norm weights, one upload
    LoraState lora;
    try {
        const std::string p0 = "layers." + std::to_string(s->first_layer);
        s->wtype = (int) f.get(p0 + ".attention.wq.weight", {E, E}).type;
        const bool kq = wt_kquant(s->wtype);
        if (!wt_block_quant(s->wtype) && s->wtype != kWT_F16 && !kq)
            return fail(B200_EFILE, "weight type %d unsupported (Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, F16, Q4_K, Q6_K): %s", s->wtype,
                        (p0 + ".attention.wq.weight").c_str());
        if (kq && (E % 256 || FF % 256))
            return fail(B200_EFILE, "k-quant slice needs n_embd and n_ff divisible by 256 (n_embd %u, n_ff %u)", E, FF);
        float * d_norms = nullptr;
        if ((rc = dev_alloc(s, &d_norms, (size_t) s->L * 2 * E))) return rc;
        norms.resize((size_t) s->L * 2 * E);
        for (int i = 0; i < s->L; i++) {
            const std::string p = "layers." + std::to_string(i + s->first_layer);
            LayerW & Lw = s->layers[i];
            const GgjtTensor & an = f.get(p + ".attention_norm.weight", {E});
            const GgjtTensor & wq = f.get(p + ".attention.wq.weight", {E, E});
            const GgjtTensor & wk = f.get(p + ".attention.wk.weight", {E, E});
            const GgjtTensor & wv = f.get(p + ".attention.wv.weight", {E, E});
            const GgjtTensor & wo = f.get(p + ".attention.wo.weight", {E, E});
            const GgjtTensor & fn = f.get(p + ".ffn_norm.weight", {E});
            const GgjtTensor & w1 = f.get(p + ".feed_forward.w1.weight", {E, FF});
            const GgjtTensor & w2 = f.get(p + ".feed_forward.w2.weight", {FF, E});
            const GgjtTensor & w3 = f.get(p + ".feed_forward.w3.weight", {E, FF});
            if (an.type != GT_F32 || fn.type != GT_F32) return fail(B200_EFILE, "norm weights must be F32");
            for (const GgjtTensor * t : {&wq, &wk, &wv, &wo, &w1, &w2, &w3}) {
                // a k-quant slice holds Q4_K and Q6_K matrices in any mix (Q4_K_S / Q4_K_M / Q6_K files)
                if (kq && !wt_kquant((int) t->type))
                    return fail(B200_EFILE, "%s has type %u: a k-quant slice takes Q4_K (12) and Q6_K (14) matrices only", t->name.c_str(), t->type);
                if (!kq && (int) t->type != s->wtype) return fail(B200_EFILE, "mixed weight types in slice (%s)", t->name.c_str());
            }
            if (kq && w1.type != w3.type)
                return fail(B200_EFILE, "%s (type %u) and %s (type %u) differ: w1 and w3 are packed together", w1.name.c_str(), w1.type,
                            w3.name.c_str(), w3.type);
            Lw.attn_norm = d_norms + (size_t) i * 2 * E; Lw.ffn_norm = Lw.attn_norm + E;
            memcpy(norms.data() + (size_t) i * 2 * E, f.data(an), (size_t) E * 4);
            memcpy(norms.data() + (size_t) i * 2 * E + E, f.data(fn), (size_t) E * 4);
            if (s->wtype == kWT_F16) {
                const GgjtTensor * ts[7] = {&wq, &wk, &wv, &wo, &w1, &w2, &w3};
                uint16_t ** dst[7] = {&Lw.f_q, &Lw.f_k, &Lw.f_v, &Lw.f_o, &Lw.f_1, &Lw.f_2, &Lw.f_3};
                const size_t per = (size_t) E * ((E / 32 + 7) / 8) * 256;          // packed elements of one E x E matrix
                uint16_t * qkv_buf = nullptr;
                if ((rc = dev_alloc(s, &qkv_buf, 3 * per + 8))) return rc;
                for (int k = 0; k < 7; k++) {
                    LoadJob j; j.kind = 1; j.nsrc = 1; j.src[0] = ts[k]; j.outf = dst[k]; j.into = k < 3 ? qkv_buf + k * per : nullptr;
                    jobs.push_back(j);
                }
            } else {
                // wq | wk | wv back to back, cut into runs of one type (only k-quant slices mix types)
                const GgjtTensor * qkv[3] = {&wq, &wk, &wv};
                for (int t0 = 0, part = 0; t0 < 3; part++) {
                    int t1 = t0 + 1;
                    while (t1 < 3 && qkv[t1]->type == qkv[t0]->type) t1++;
                    LoadJob a; a.nsrc = t1 - t0; a.mode = a.nsrc > 1 ? 1 : 0; a.G = 1;
                    for (int k = t0; k < t1; k++) a.src[k - t0] = qkv[k];
                    a.out = part == 0 ? &Lw.qkv : &Lw.qkv_more[part - 1];
                    if (part > 0) Lw.qkv_row[part - 1] = t0 * (int) E;
                    jobs.push_back(a);
                    t0 = t1;
                }
                LoadJob o; o.nsrc = 1; o.src[0] = &wo; o.mode = 0; o.G = 1; o.out = &Lw.wo;
                jobs.push_back(o);
                LoadJob g; g.nsrc = 2; g.src[0] = &w1; g.src[1] = &w3; g.mode = 2; g.G = 2; g.out = &Lw.w13; jobs.push_back(g);
                LoadJob d; d.nsrc = 1; d.src[0] = &w2; d.mode = 0; d.G = 1; d.out = &Lw.w2;
                jobs.push_back(d);
            }
            s->weight_bytes += (int64_t)(an.nbytes + fn.nbytes + wq.nbytes + wk.nbytes + wv.nbytes + wo.nbytes + w1.nbytes + w2.nbytes + w3.nbytes);
        }
        B200_CUDA(cudaMemcpyAsync(d_norms, norms.data(), norms.size() * 4, cudaMemcpyHostToDevice, s->stream));
        if (lora_path && (rc = plan_lora(s, f, lora_path, base_path, jobs, lora))) return rc;
        if ((rc = run_load_jobs(s, f, jobs, lora.merge))) return rc;
    } catch (const std::exception & e) {
        return fail(B200_EFILE, "error loading model: %s", e.what());
    }
    lap("weights: read + upload + repack");

    const size_t nE = (size_t) s->n_ctx * E;
    s->sess_stride = (size_t) s->L * nE;
    s->past.assign(s->n_sessions, 0);
    if ((rc = dev_alloc(s, &s->kc, s->n_sessions * s->sess_stride)) || (rc = dev_alloc(s, &s->vc, s->n_sessions * s->sess_stride)) ||
        (rc = dev_alloc(s, &s->d_pass, pass_table_ints(s->n_ctx, s->n_sessions))) ||
        (rc = dev_alloc(s, &s->q16, nE)) || (rc = dev_alloc(s, &s->xa, nE)) || (rc = dev_alloc(s, &s->xb, nE)) ||
        (rc = dev_alloc(s, &s->qkv, 3 * nE)) || (rc = dev_alloc(s, &s->att, nE)) || (rc = dev_alloc(s, &s->ffin, nE)) ||
        (rc = dev_alloc(s, &s->gate, (size_t) s->n_ctx * FF)) || (rc = dev_alloc(s, &s->d_in, nE)) ||
        (rc = dev_alloc(s, &s->d_out, nE)) || (rc = dev_alloc(s, &s->d_npast, (size_t) s->n_sessions)) ||
        (rc = dev_alloc(s, &s->d_kvdst, (size_t) s->n_sessions)))
        return rc;
    if ((rc = dev_alloc(s, &s->xh, (size_t) s->n_ctx * (FF > E ? FF : E) + 64))) return rc;
    if (wt_kquant(s->wtype)) {
        const int nbq = std::max(s->layers[0].wo.nbq, s->layers[0].w2.nbq);   // K = n_embd and K = n_ff
        if ((rc = dev_alloc(s, &s->kq_aq, (size_t) s->n_ctx * nbq * 72)) || (rc = dev_alloc(s, &s->kq_ad, (size_t) s->n_ctx * kq_nbd(nbq))))
            return rc;
    }
    if (s->wtype != kWT_F16 && !wt_kquant(s->wtype)) {
        s->nbqE = s->layers[0].wo.nbq; s->nbqF = s->layers[0].w2.nbq;
        const size_t nq = (size_t) s->n_ctx;
        // Q4_1 / Q5_1: every scale array carries a second plane (Q8_1's block sums s) right behind the scales
        const size_t pl = wt_q8_1(s->wtype) ? 2 : 1;
        if (pl == 2) { s->soffE = (int)(nq * s->nbqE * 4); s->soffF = (int)(nq * s->nbqF * 4); }
        if ((rc = dev_alloc(s, &s->aq_att, nq * s->nbqE * 32)) || (rc = dev_alloc(s, &s->da_att, pl * nq * s->nbqE * 4)) ||
            (rc = dev_alloc(s, &s->aq_gate, nq * s->nbqF * 32)) || (rc = dev_alloc(s, &s->da_gate, pl * nq * s->nbqF * 4))) return rc;
        if ((rc = dev_alloc(s, &s->aq_x, nq * s->nbqE * 32)) || (rc = dev_alloc(s, &s->da_x, pl * nq * s->nbqE * 4)) ||
            (rc = dev_alloc(s, &s->nq_counter, 2 * nq)) || (rc = dev_alloc(s, &s->nq_partial, nq * 256))) return rc;
        B200_CUDA(cudaMemset(s->aq_x, 0, nq * s->nbqE * 128)); B200_CUDA(cudaMemset(s->da_x, 0, pl * nq * s->nbqE * 16));
        B200_CUDA(cudaMemset(s->nq_counter, 0, 2 * nq * 4));
        B200_CUDA(cudaMemset(s->aq_att, 0, nq * s->nbqE * 128));  B200_CUDA(cudaMemset(s->da_att, 0, pl * nq * s->nbqE * 16));
        B200_CUDA(cudaMemset(s->aq_gate, 0, nq * s->nbqF * 128)); B200_CUDA(cudaMemset(s->da_gate, 0, pl * nq * s->nbqF * 16));
    }
    B200_CUDA(cudaMemset(s->kc, 0, s->n_sessions * s->sess_stride * 2));
    B200_CUDA(cudaMemset(s->vc, 0, s->n_sessions * s->sess_stride * 2));
    B200_CUDA(cudaMemset(s->d_npast, 0, 4 * (size_t) s->n_sessions));
    B200_CUDA(cudaMallocHost((void **) &s->h_in, (size_t) E * 4));
    B200_CUDA(cudaMallocHost((void **) &s->h_out, (size_t) E * 4));
    lap("KV cache + activations");
    if ((rc = build_tables(s))) return rc;
    lap("exp / SiLU / RoPE tables");
    if (env_int("B200_TRACE", 0)) {
        if ((rc = dev_alloc(s, &s->trace, (size_t) 512 * 1024 * 8))) return rc;
        B200_CUDA(cudaMemset(s->trace, 0, (size_t) 512 * 1024 * 8 * 8));
    }
    B200_CUDA(cudaFuncSetAttribute(k_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    B200_CUDA(cudaFuncSetAttribute(k_attn128<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    B200_CUDA(cudaFuncSetAttribute(k_attn128<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    if (s->D == 128) {
        // The single-token attention runs one 4-CTA cluster per head, and each cluster can start only on four free SMs of
        // one GPC.  With the exp table's 64 KB staged in shared memory a CTA takes most of an SM, and a device may hold
        // fewer clusters than there are heads (H100 SXM, 7B: 30 of 32): the rest wait for a whole second wave, every
        // layer.  Then the table is read through L2 instead (the same entries, so the same results).
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(4 * s->H, 1, 1); cfg.blockDim = dim3(256, 1, 1); cfg.dynamicSmemBytes = attn_need;
        int clusters = 0;
        B200_CUDA(cudaOccupancyMaxActiveClusters(&clusters, k_attn128<true>, &cfg));
        s->attn_lut_smem = clusters >= s->H;
        if (ltrace) fprintf(stderr, "[b200 load] single-token attention: %d of %d clusters resident with the exp table in shared memory: %s\n",
                            clusters, s->H, s->attn_lut_smem ? "staged" : "read through L2");
    }
    B200_CUDA(cudaEventCreate(&s->ev0));
    B200_CUDA(cudaEventCreate(&s->ev1));
    B200_CUDA(cudaDeviceSynchronize());
    lap("attributes + final sync");
    if (ltrace) fprintf(stderr, "[b200 load] total %.3f s for %.2f GB of weights\n", tnow() - t_begin, s->weight_bytes / 1e9);
    return 0;
}

static void destroy(b200_slice * s) {
    cudaSetDevice(s->device);
    if (s->stream) cudaStreamSynchronize(s->stream);
    for (auto & kv : s->graphs) cudaGraphExecDestroy(kv.second);
    for (auto & kv : s->pp_graphs) cudaGraphExecDestroy(kv.second);
    if (s->mb_next) cudaIpcCloseMemHandle(s->mb_next);
    if (s->mb_prev && s->mb_prev != s->mb_next) cudaIpcCloseMemHandle(s->mb_prev);
    for (void * p : s->allocs) cudaFree(p);
    if (s->h_in) cudaFreeHost(s->h_in);
    if (s->h_out) cudaFreeHost(s->h_out);
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    for (cudaEvent_t e : s->prof_ev) cudaEventDestroy(e);
    for (int i = 0; i < 2; i++) if (s->mark[i]) cudaEventDestroy(s->mark[i]);
    if (s->stream) cudaStreamDestroy(s->stream);
    delete s;
}

// Session src's cache rows [0, n_keep) to each of dsts[0, n_dst) (distinct, none equal to src; the caller checked), and the
// destinations' positions to n_keep: host copy now, device copy in order on cs.  A destination's rows at or above n_keep
// keep their bytes; nothing reads them before it writes them again (attention reads rows below the session's position).
static int kv_fork(b200_slice * s, int src, const int * dsts, int n_dst, int n_keep, cudaStream_t cs) {
    if (n_keep > 0) {
        B200_CUDA(cudaMemcpyAsync(s->d_kvdst, dsts, 4 * (size_t) n_dst, cudaMemcpyHostToDevice, cs));
        if (int rc = smem_attr<k_kv_fanout>(s, kFanSmem)) return rc;
        const uint32_t plane = (uint32_t) n_keep * s->E * 2, n_chunks = (plane + kFanChunk - 1) / kFanChunk;
        const int planes = 2 * s->L;
        // about three CTAs per SM (64 KB of stages each), so a few loads and every destination's stores are in flight
        const uint32_t per_plane = std::min<uint32_t>(n_chunks, (uint32_t) std::max(1, (3 * s->n_sm + planes - 1) / planes));
        k_kv_fanout<<<dim3(per_plane, planes), 32, kFanSmem, cs>>>(s->kc, s->vc, s->sess_stride, (size_t) s->n_ctx * s->E, src,
                                                                    s->d_kvdst, n_dst, plane);
        B200_CUDA(cudaGetLastError());
        s->launches++;
    }
    for (int d = 0; d < n_dst; d++) {
        B200_CUDA(cudaMemcpyAsync(s->d_npast + dsts[d], &n_keep, 4, cudaMemcpyHostToDevice, cs));
        s->past[dsts[d]] = n_keep;
    }
    return 0;
}

// A handle inside an open generation stream belongs to it: a call from elsewhere fails at once instead of waiting for the
// stream to end or racing the steps it has enqueued.
static int refuse_owned(const b200_slice * s) {
    return fail(B200_EINVAL, "the handle belongs to the open generation stream %p: b200_stream_close it first", (const void *) s->owner);
}
#define B200_UNOWNED(h) do { if ((h)->owner) return b200::refuse_owned(h); } while (0)

}  // namespace b200

// ============================================================================ C ABI
extern "C" {

const char * b200_last_error(void) { return b200::last_error_ref().c_str(); }
const char * b200_version(void) { return "b200-slice 0.1 (sm_90a, exact mode)"; }

int b200_slice_load(const char * path, int device, int n_ctx, b200_slice_t ** out) {
    return b200_slice_load_ex(path, device, n_ctx, 1, out);
}

int b200_slice_load_ex(const char * path, int device, int n_ctx, int n_sessions, b200_slice_t ** out) {
    return b200_slice_load_lora(path, device, n_ctx, n_sessions, nullptr, nullptr, out);
}

int b200_slice_load_lora(const char * path, int device, int n_ctx, int n_sessions, const char * lora_path,
                         const char * lora_base_path, b200_slice_t ** out) {
    if (!path || !out) return fail(B200_EINVAL, "b200_slice_load: null argument");
    if (lora_base_path && !lora_path) return fail(B200_EINVAL, "b200_slice_load_lora: a LoRA base without an adapter");
    *out = nullptr;
    if (n_sessions < 1 || n_sessions > 4096) return fail(B200_EINVAL, "n_sessions %d outside [1, 4096]", n_sessions);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(B200_ENODEV, "no CUDA device visible: the slice forward has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(B200_ENODEV, "device %d out of range (%d visible)", device, ndev);
    cudaDeviceProp prop;
    B200_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(B200_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    B200_CUDA(cudaSetDevice(device));
    b200_slice * s = new b200_slice();
    s->device = device; s->n_sm = prop.multiProcessorCount;
    s->n_ctx = n_ctx > 0 ? n_ctx : 512;               // vendor examples/common.h:28
    s->n_sessions = n_sessions;
    s->use_ring  = env_int("B200_RING", 1) != 0;
    s->use_graph = env_int("B200_GRAPH", 1) != 0;
    s->use_pdl   = env_int("B200_PDL", 1) != 0;
    s->fast_prefill = env_int("B200_FAST_PREFILL", 0) != 0; s->fast_min_tokens = env_int("B200_FAST_MIN_TOKENS", 32);
    s->use_nq    = env_int("B200_NQ", 0) != 0;   // grid-barrier norm+quant epilogue in wo / w2 (decode): exact, opt-in (its barrier costs what it saves)
    s->opt_ns = env_int("B200_NS", 0); s->opt_cta_per_sm = env_int("B200_CTA_PER_SM", 0); s->opt_nc = env_int("B200_NC", 0);
    s->opt_pre = env_int("B200_PRE", 3); s->opt_nomath = env_int("B200_DBG_NOMATH", 0);
    s->use_tiled_attn = env_int("B200_TILED_ATTN", 1) != 0;   // prompt chunks: query-tiled attention (K / V staged once per 16 queries)
    s->f16_mc = env_int("B200_F16_MC", 1) != 0;      // F16 slices, multi-token calls: 4 (8) columns per CTA share the weight loads
    s->f16_mc_cols = env_int("B200_F16_MC", 1) == 8 ? 8 : 4;
    s->f16_ring = env_int("B200_F16_RING", 1) != 0;          // F16-weight slices: TMA-ring matmul for single-token steps
    cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { delete s; return fail(B200_ECUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e)); }
    int rc = load_locked(s, path, lora_path, lora_base_path);
    if (rc) { destroy(s); return rc; }
    *out = s;
    return 0;
}

int b200_slice_unload(b200_slice_t * s) {
    if (!s) return fail(B200_EINVAL, "null handle");
    { std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s); }   // let a call that is inside the library finish (see the header: no NEW call may race unload)
    destroy(s);
    return 0;
}

/* Create the CUDA context of `device` (cudaSetDevice + a no-op runtime call).  The first CUDA call of a process costs
 * 0.3 s on a 1-GPU box and several seconds on an 8-GPU box; callers that time b200_slice_load can pay it up front. */
int b200_device_init(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(B200_ENODEV, "no CUDA device visible: the slice forward has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(B200_ENODEV, "device %d out of range (%d visible)", device, ndev);
    B200_CUDA(cudaSetDevice(device));
    B200_CUDA(cudaFree(nullptr));
    return 0;
}

int b200_slice_clear(b200_slice_t * s) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaMemsetAsync(s->d_npast, 0, 4, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->past[0] = 0;
    return 0;
}

int b200_slice_rewind(b200_slice_t * s, int n_past) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (n_past < 0 || n_past > s->past[0]) return fail(B200_EINVAL, "rewind target %d outside [0, %d]", n_past, s->past[0]);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaMemcpyAsync(s->d_npast, &n_past, 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->past[0] = n_past;
    return 0;
}

int b200_slice_info(b200_slice_t * s, b200_slice_info_t * info) {
    if (!s || !info) return fail(B200_EINVAL, "null argument");
    B200_UNOWNED(s);
    info->n_embd = s->E; info->n_head = s->H; info->n_ff = s->FF; info->n_layer = s->L; info->first_layer = s->first_layer;
    info->n_ctx = s->n_ctx; info->n_past = s->past[0]; info->weight_type = s->wtype; info->device = s->device;
    info->weight_bytes = s->weight_bytes; info->kv_bytes_per_pos = (int64_t) s->L * 2 * s->E * 2;
    return 0;
}

int b200_slice_forward(b200_slice_t * s, const float * in, int n_tokens, float * out) {
    if (!s || !in || !out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return forward_locked(s, in, n_tokens, out, true);
}

int b200_slice_forward_device(b200_slice_t * s, const float * d_in, int n_tokens, float * d_out, int sync) {
    if (!s || !d_in || !d_out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    int rc = forward_locked(s, d_in, n_tokens, d_out, false);
    if (rc) return rc;
    if (sync) B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

/* ---- sessions and batched steps (additive; SURVEY 8f N3) ---- */
int b200_session_count(b200_slice_t * s) { return s ? s->n_sessions : 0; }

int b200_session_n_past(b200_slice_t * s, int session) {
    if (!s || session < 0 || session >= s->n_sessions) return -1;
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->owner) { refuse_owned(s); return -1; }
    return s->past[session];
}

int b200_session_clear(b200_slice_t * s, int session) {
    if (!s) return fail(B200_EINVAL, "null handle");
    if (session < -1 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    if (session < 0) {
        B200_CUDA(cudaMemsetAsync(s->d_npast, 0, 4 * (size_t) s->n_sessions, s->stream));
        std::fill(s->past.begin(), s->past.end(), 0);
    } else {
        B200_CUDA(cudaMemsetAsync(s->d_npast + session, 0, 4, s->stream));
        s->past[session] = 0;
    }
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_session_rewind(b200_slice_t * s, int session, int n_past) {
    if (!s) return fail(B200_EINVAL, "null handle");
    if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (n_past < 0 || n_past > s->past[session]) return fail(B200_EINVAL, "rewind target %d outside [0, %d]", n_past, s->past[session]);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaMemcpyAsync(s->d_npast + session, &n_past, 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->past[session] = n_past;
    return 0;
}

int b200_session_copy(b200_slice_t * s, int src, const int * dsts, int n_dst, int n_keep) {
    if (!s || !dsts) return fail(B200_EINVAL, "b200_session_copy: null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (n_dst < 1) return fail(B200_EINVAL, "b200_session_copy: n_dst must be positive (got %d)", n_dst);
    if (src < 0 || src >= s->n_sessions) return fail(B200_EINVAL, "source session %d outside [0, %d)", src, s->n_sessions);
    std::vector<char> seen(s->n_sessions, 0);
    for (int d = 0; d < n_dst; d++) {
        const int k = dsts[d];
        if (k < 0 || k >= s->n_sessions) return fail(B200_EINVAL, "destination %d is session %d, outside [0, %d)", d, k, s->n_sessions);
        if (k == src) return fail(B200_EINVAL, "destination %d is the source session %d", d, src);
        if (seen[k]++) return fail(B200_EINVAL, "session %d is listed twice as a destination", k);
    }
    if (n_keep < 0 || n_keep > s->past[src])
        return fail(B200_EINVAL, "n_keep %d outside [0, %d] (the source's position)", n_keep, s->past[src]);
    B200_CUDA(cudaSetDevice(s->device));
    if (int rc = kv_fork(s, src, dsts, n_dst, n_keep, s->stream)) return rc;
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

/* Session state blob: a 64-byte little-endian header, then K rows [layer][n_past][n_embd] fp16, then V rows alike. */
namespace {
constexpr size_t kStateHeader = 64;
constexpr uint32_t kStateVersion = 1;
enum { kHdrMagic = 0, kHdrVersion = 4, kHdrEmbd = 8, kHdrHead = 12, kHdrLayer = 16, kHdrFirst = 20, kHdrPast = 24 };
void put_u32(uint8_t * p, uint32_t v) { for (int i = 0; i < 4; i++) p[i] = (uint8_t) (v >> (8 * i)); }
uint32_t get_u32(const uint8_t * p) { uint32_t v = 0; for (int i = 0; i < 4; i++) v |= (uint32_t) p[i] << (8 * i); return v; }
size_t state_bytes(const b200_slice * s, int n_past) { return kStateHeader + (size_t) n_past * s->L * 2 * s->E * 2; }
}  // namespace

int b200_session_state_size(b200_slice_t * s, int session, size_t * bytes) {
    if (!s || !bytes) return fail(B200_EINVAL, "b200_session_state_size: null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    *bytes = state_bytes(s, s->past[session]);
    return 0;
}

int b200_session_save(b200_slice_t * s, int session, void * buf, size_t cap, size_t * written) {
    if (!s || !buf) return fail(B200_EINVAL, "b200_session_save: null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    const int n_past = s->past[session];
    const size_t need = state_bytes(s, n_past);
    if (cap < need) return fail(B200_EINVAL, "b200_session_save: the buffer holds %zu bytes, the state needs %zu", cap, need);
    uint8_t * h = (uint8_t *) buf;
    memset(h, 0, kStateHeader);
    memcpy(h + kHdrMagic, "B2KV", 4);
    put_u32(h + kHdrVersion, kStateVersion); put_u32(h + kHdrEmbd, s->E); put_u32(h + kHdrHead, s->H);
    put_u32(h + kHdrLayer, s->L); put_u32(h + kHdrFirst, s->first_layer); put_u32(h + kHdrPast, n_past);
    const size_t row = (size_t) n_past * s->E * 2, pitch = (size_t) s->n_ctx * s->E * 2;
    B200_CUDA(cudaSetDevice(s->device));
    if (row) {
        B200_CUDA(cudaMemcpy2DAsync(h + kStateHeader, row, s->kc + session * s->sess_stride, pitch, row, s->L, cudaMemcpyDeviceToHost, s->stream));
        B200_CUDA(cudaMemcpy2DAsync(h + kStateHeader + row * s->L, row, s->vc + session * s->sess_stride, pitch, row, s->L,
                                    cudaMemcpyDeviceToHost, s->stream));
    }
    B200_CUDA(cudaStreamSynchronize(s->stream));
    if (written) *written = need;
    return 0;
}

int b200_session_restore(b200_slice_t * s, int session, const void * buf, size_t n) {
    if (!s || !buf) return fail(B200_EINVAL, "b200_session_restore: null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
    const uint8_t * h = (const uint8_t *) buf;
    if (n < kStateHeader || memcmp(h + kHdrMagic, "B2KV", 4) != 0) return fail(B200_EINVAL, "b200_session_restore: not a session state");
    if (get_u32(h + kHdrVersion) != kStateVersion)
        return fail(B200_EINVAL, "b200_session_restore: state version %u, this library reads %u", get_u32(h + kHdrVersion), kStateVersion);
    const int E = (int) get_u32(h + kHdrEmbd), H = (int) get_u32(h + kHdrHead), L = (int) get_u32(h + kHdrLayer),
              first = (int) get_u32(h + kHdrFirst), n_past = (int) get_u32(h + kHdrPast);
    if (E != s->E || H != s->H || L != s->L || first != s->first_layer)
        return fail(B200_EINVAL, "b200_session_restore: the state is of n_embd %d, n_head %d, layers %d..%d; the slice of %d, %d, %d..%d",
                    E, H, first, first + L - 1, s->E, s->H, s->first_layer, s->first_layer + s->L - 1);
    if (n_past < 0 || n_past > s->n_ctx) return fail(B200_EINVAL, "b200_session_restore: n_past %d outside [0, n_ctx %d]", n_past, s->n_ctx);
    if (n != state_bytes(s, n_past))
        return fail(B200_EINVAL, "b200_session_restore: %zu bytes, a state of %d positions has %zu", n, n_past, state_bytes(s, n_past));
    const size_t row = (size_t) n_past * s->E * 2, pitch = (size_t) s->n_ctx * s->E * 2;
    B200_CUDA(cudaSetDevice(s->device));
    if (row) {
        B200_CUDA(cudaMemcpy2DAsync(s->kc + session * s->sess_stride, pitch, h + kStateHeader, row, row, s->L, cudaMemcpyHostToDevice, s->stream));
        B200_CUDA(cudaMemcpy2DAsync(s->vc + session * s->sess_stride, pitch, h + kStateHeader + row * s->L, row, row, s->L,
                                    cudaMemcpyHostToDevice, s->stream));
    }
    B200_CUDA(cudaMemcpyAsync(s->d_npast + session, &n_past, 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->past[session] = n_past;
    return 0;
}

int b200_session_forward(b200_slice_t * s, int session, const float * in, int n_tokens, float * out) {
    if (!s || !in || !out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return forward_locked(s, in, n_tokens, out, true, session);
}

int b200_session_forward_device(b200_slice_t * s, int session, const float * d_in, int n_tokens, float * d_out, int sync) {
    if (!s || !d_in || !d_out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    int rc = forward_locked(s, d_in, n_tokens, d_out, false, session);
    if (rc) return rc;
    if (sync) B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_session_forward_steps(b200_slice_t * s, int session, const float * in, int n_tokens, float * out) {
    if (!s || !in || !out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return steps_locked(s, session, in, n_tokens, out, true);
}

int b200_session_forward_steps_device(b200_slice_t * s, int session, const float * d_in, int n_tokens, float * d_out, int sync) {
    if (!s || !d_in || !d_out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    int rc = steps_locked(s, session, d_in, n_tokens, d_out, false);
    if (rc) return rc;
    if (sync) B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_batch_forward(b200_slice_t * s, const int * sessions, int n_seq, const float * in, float * out) {
    if (!s || !sessions || !in || !out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return pass_locked(s, sessions, nullptr, n_seq, in, out, true);
}

int b200_batch_forward_device(b200_slice_t * s, const int * sessions, int n_seq, const float * d_in, float * d_out, int sync) {
    if (!s || !sessions || !d_in || !d_out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    int rc = pass_locked(s, sessions, nullptr, n_seq, d_in, d_out, false);
    if (rc) return rc;
    if (sync) B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_mixed_forward(b200_slice_t * s, const int * sessions, const int * counts, int n_seq, const float * in, float * out) {
    if (!s || !sessions || !counts || !in || !out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return pass_locked(s, sessions, counts, n_seq, in, out, true);
}

int b200_mixed_forward_device(b200_slice_t * s, const int * sessions, const int * counts, int n_seq, const float * d_in, float * d_out, int sync) {
    if (!s || !sessions || !counts || !d_in || !d_out) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    int rc = pass_locked(s, sessions, counts, n_seq, d_in, d_out, false);
    if (rc) return rc;
    if (sync) B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_slice_sync(b200_slice_t * s) {
    if (!s) return fail(B200_EINVAL, "null handle");
    B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

float b200_slice_last_ms(b200_slice_t * s) {
    if (!s || !s->timed) return -1.f;
    float ms = -1.f;
    cudaSetDevice(s->device);
    if (cudaEventSynchronize(s->ev1) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) != cudaSuccess) return -1.f;
    return ms;
}

int64_t b200_slice_launch_count(b200_slice_t * s) { return s ? s->launches : 0; }
float * b200_slice_dev_in(b200_slice_t * s)  { return s ? s->d_in : nullptr; }
float * b200_slice_dev_out(b200_slice_t * s) { return s ? s->d_out : nullptr; }

int b200_slice_set_fast_prefill(b200_slice_t * s, int on, int min_tokens) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    s->fast_prefill = on != 0;
    if (min_tokens > 0) s->fast_min_tokens = min_tokens;
    return 0;
}

/* Measurement aid for bench.py's roofline: while on, a decode step launches ONLY its weight-matmul kernels (the
 * attention launch is skipped, so hidden states are meaningless and the KV cache is not appended). */
int b200_debug_skip_attention(b200_slice_t * s, int on) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    s->skip_attention = on != 0;
    return 0;
}

int b200_slice_mark(b200_slice_t * s, int which) {
    if (!s || which < 0 || which > 1) return fail(B200_EINVAL, "bad argument");
    B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    if (!s->mark[which]) B200_CUDA(cudaEventCreate(&s->mark[which]));
    B200_CUDA(cudaEventRecord(s->mark[which], s->stream));
    return 0;
}

float b200_slice_mark_elapsed_ms(b200_slice_t * s) {
    if (!s || !s->mark[0] || !s->mark[1]) return -1.f;
    float ms = -1.f;
    cudaSetDevice(s->device);
    if (cudaEventSynchronize(s->mark[1]) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, s->mark[0], s->mark[1]) != cudaSuccess) return -1.f;
    return ms;
}

int b200_slice_profile(b200_slice_t * s, int enable) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    s->profiling = enable != 0; s->prof_used = 0; s->prof_cls.clear();
    return 0;
}

int b200_slice_profile_read(b200_slice_t * s, float * ms_by_class, int * launches_by_class, int n_class) {
    if (!s || !ms_by_class || !launches_by_class) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    for (int i = 0; i < n_class; i++) { ms_by_class[i] = 0.f; launches_by_class[i] = 0; }
    for (size_t i = 0; i < s->prof_cls.size(); i++) {
        float ms = 0.f;
        B200_CUDA(cudaEventElapsedTime(&ms, s->prof_ev[2 * i], s->prof_ev[2 * i + 1]));
        const int c = s->prof_cls[i];
        if (c < n_class) { ms_by_class[c] += ms; launches_by_class[c]++; }
    }
    s->prof_used = 0; s->prof_cls.clear();
    return 0;
}

/* Switch the in-kernel timeline on or off at run time (drops the captured decode graphs so the next step re-captures). */
int b200_debug_trace_enable(b200_slice_t * s, int on) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    for (auto & kv : s->graphs) cudaGraphExecDestroy(kv.second);
    s->graphs.clear();
    static unsigned long long * parked = nullptr;
    if (on) {
        if (!s->trace) {
            if (parked) { s->trace = parked; parked = nullptr; }
            else { int rc = dev_alloc(s, &s->trace, (size_t) 512 * 1024 * 8); if (rc) return rc; }
        }
        B200_CUDA(cudaMemset(s->trace, 0, (size_t) 512 * 1024 * 8 * 8));
        s->trace_next = 0; s->trace_cls.clear(); s->trace_ctas.clear();
    } else if (s->trace) { parked = s->trace; s->trace = nullptr; }
    return 0;
}

/* Debug timeline: when B200_TRACE=1 every matmul / attention launch of the NEXT captured graph (or un-graphed step)
 * stamps %globaltimer per CTA: [0] entry, [1] after griddepcontrol.wait, [2] prologue done, [3] exit, [4] last weight copy issued. */
int b200_debug_trace_read(b200_slice_t * s, unsigned long long * out, int * cls, int * ctas, int max_launches) {
    if (!s || !s->trace) return 0;
    cudaSetDevice(s->device);
    cudaStreamSynchronize(s->stream);
    int n = s->trace_next < max_launches ? s->trace_next : max_launches;
    cudaMemcpy(out, s->trace, (size_t) n * 1024 * 8 * 8, cudaMemcpyDeviceToHost);
    for (int i = 0; i < n; i++) { cls[i] = s->trace_cls[i]; ctas[i] = s->trace_ctas[i]; }
    return n;
}

/* Test hook: copy `count` 32-bit words of an internal activation buffer to the host after a
 * forward (0 qkv, 1 att, 2 ffin, 3 gate, 4 xa, 5 xb, 6 q16, 7 k-cache, 8 v-cache, 9 xh: the fp16 activations of the
 * last fast-mode matmul, 10 the slice's output staging buffer d_out). */
int b200_debug_read(b200_slice_t * s, int which, size_t offset_words, size_t count, void * out) {
    if (!s || !out) return fail(B200_EINVAL, "null argument");
    B200_UNOWNED(s);
    const void * src[11] = {s->qkv, s->att, s->ffin, s->gate, s->xa, s->xb, s->q16, s->kc, s->vc, s->xh, s->d_out};
    if (which < 0 || which > 10) return fail(B200_EINVAL, "bad buffer id %d", which);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    B200_CUDA(cudaMemcpy(out, (const uint32_t *) src[which] + offset_words, count * 4, cudaMemcpyDeviceToHost));
    return 0;
}

/* Test hook: the packed bytes of one weight matrix of layer `layer` (0 = the slice's first).  Block-quantised and
 * k-quant slices: which 0 qkv, 1 wo, 2 w13, 3 w2, 4 / 5 the second / third qkv run of a k-quant slice; F16 slices:
 * which 0..6 = wq, wk, wv, wo, w1, w2, w3.  k_repack / k_repack_kq write every word of n_tiles * tile_bytes and
 * k_repack_f16 every element of rows * nc8 * 256 (padding as zeros), so two loads of equal source bytes give equal
 * bytes here.  *size (if not null) receives the matrix's byte count; `count` bytes from `offset` are copied to out. */
int b200_debug_weights(b200_slice_t * s, int layer, int which, size_t offset, size_t count, void * out, size_t * size) {
    if (!s) return fail(B200_EINVAL, "null handle");
    B200_UNOWNED(s);
    if (layer < 0 || layer >= s->L) return fail(B200_EINVAL, "layer %d outside [0, %d)", layer, s->L);
    const LayerW & Lw = s->layers[layer];
    const void * src = nullptr;
    size_t n = 0;
    if (s->wtype == kWT_F16) {
        if (which < 0 || which > 6) return fail(B200_EINVAL, "bad F16 matrix id %d (0..6: wq wk wv wo w1 w2 w3)", which);
        const uint16_t * f[7] = {Lw.f_q, Lw.f_k, Lw.f_v, Lw.f_o, Lw.f_1, Lw.f_2, Lw.f_3};
        const int rows = which == 4 || which == 6 ? s->FF : s->E, K = which == 5 ? s->FF : s->E;
        src = f[which];
        n = (size_t) rows * ((K / 32 + 7) / 8) * 256 * 2;
    } else {
        if (which < 0 || which > 5) return fail(B200_EINVAL, "bad matrix id %d (0..5: qkv wo w13 w2 qkv_more[0..1])", which);
        const PackedW * w[6] = {&Lw.qkv, &Lw.wo, &Lw.w13, &Lw.w2, &Lw.qkv_more[0], &Lw.qkv_more[1]};
        src = w[which]->data;
        n = src ? (size_t) w[which]->n_tiles * (size_t) w[which]->tile_bytes : 0;
    }
    if (size) *size = n;
    if (!count) return 0;
    if (!out) return fail(B200_EINVAL, "null argument");
    if (offset > n || count > n - offset) return fail(B200_EINVAL, "bytes [%zu, %zu) outside the matrix's %zu", offset, offset + count, n);
    B200_CUDA(cudaSetDevice(s->device));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    B200_CUDA(cudaMemcpy(out, (const uint8_t *) src + offset, count, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"


// ============================================================================ layer-slice pipeline (NCCL)
// The reference relays the activation between nodes through the client over TCP, one request per hop
// (cli_api/common.py:148-154 -> control_center.py:224-244 -> routes.py:176-195).  For slices that live on the
// GPUs of one NVSwitch box the hop is ONE ncclSend / ncclRecv of [n_tokens][n_embd] f32 on the slice's stream.
// NCCL is bound at run time (dlopen) so that the single-GPU path carries no dependency on it.
namespace b200 {
struct NcclId { char bytes[128]; };
struct NcclApi {
    void * lib = nullptr;
    int (*GetUniqueId)(NcclId *) = nullptr;
    int (*CommInitRank)(void **, int, NcclId, int) = nullptr;
    int (*Send)(const void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*Recv)(void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    const char * (*GetErrorString)(int) = nullptr;
};
static NcclApi & nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char * env = getenv("B200_NCCL_LIB");
        const char * names[] = {env, "libnccl.so.2", "libnccl.so"};
        for (const char * n : names) {
            if (!n) continue;
            api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) return;
        api.GetUniqueId    = (int (*)(NcclId *)) dlsym(api.lib, "ncclGetUniqueId");
        api.CommInitRank   = (int (*)(void **, int, NcclId, int)) dlsym(api.lib, "ncclCommInitRank");
        api.Send           = (int (*)(const void *, size_t, int, int, void *, cudaStream_t)) dlsym(api.lib, "ncclSend");
        api.Recv           = (int (*)(void *, size_t, int, int, void *, cudaStream_t)) dlsym(api.lib, "ncclRecv");
        api.CommDestroy    = (int (*)(void *)) dlsym(api.lib, "ncclCommDestroy");
        api.GetErrorString = (const char * (*)(int)) dlsym(api.lib, "ncclGetErrorString");
    });
    return api;
}
static int nccl_fail(const char * what, int rc) {
    NcclApi & n = nccl();
    return fail(B200_ENCCL, "%s failed: %s", what, n.GetErrorString ? n.GetErrorString(rc) : "NCCL error");
}
constexpr int kNcclFloat32 = 7;
}  // namespace b200

extern "C" {

int b200_pipeline_unique_id(void * id128) {
    NcclApi & n = nccl();
    if (!n.lib || !n.GetUniqueId) return fail(B200_ENCCL, "libnccl.so.2 not found (set B200_NCCL_LIB)");
    if (!id128) return fail(B200_EINVAL, "null id buffer");
    NcclId id;
    int rc = n.GetUniqueId(&id);
    if (rc) return nccl_fail("ncclGetUniqueId", rc);
    memcpy(id128, id.bytes, 128);
    return 0;
}

int b200_pipeline_init(b200_slice_t * s, int rank, int nranks, const void * id128) {
    if (!s || !id128 || rank < 0 || rank >= nranks) return fail(B200_EINVAL, "bad pipeline arguments");
    NcclApi & n = nccl();
    if (!n.lib || !n.CommInitRank) return fail(B200_ENCCL, "libnccl.so.2 not found (set B200_NCCL_LIB)");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    NcclId id; memcpy(id.bytes, id128, 128);
    int rc = n.CommInitRank(&s->nccl_comm, nranks, id, rank);
    if (rc) return nccl_fail("ncclCommInitRank", rc);
    s->pp_rank = rank; s->pp_world = nranks;
    if (rank == 0 && !s->d_final) { int e = dev_alloc(s, &s->d_final, (size_t) s->n_ctx * s->E); if (e) return e; }
    return 0;
}

// Peer-memory variant of a pipeline step (see kernels.cuh, "Inter-slice hand-off through PEER MEMORY"): the hop is a
// store into the next rank's mailbox + a flag, issued by k_peer_send right behind this slice's last matmul and picked
// up by k_peer_recv in front of the next slice's first matmul.  For a single-token step the whole sequence
// [recv ->] layers -> send [-> recv of the ring result] is ONE captured graph per rank: no host code between slices.
static int pipeline_step_peer(b200_slice * s, const float * d_in, int n_rows, int ring, int session, const int * sessions,
                              const int * counts, int n_seq) {
    const int r = s->pp_rank, W = s->pp_world;
    const size_t count = (size_t) n_rows * s->E;
    if (count > s->mb_slot_floats) return fail(B200_EINVAL, "hand-off of %zu floats exceeds the mailbox slot (%zu)", count, s->mb_slot_floats);
    const bool recv_in = r > 0, sends = r < W - 1 || ring, recv_final = r == 0 && ring == 1;   // ring 2: rank 0 collects later
    MailboxHdr * mine = (MailboxHdr *) s->mb_block;
    const uint2 * inbox = (const uint2 *)(s->mb_block + sizeof(MailboxHdr));
    PeerRecvArgs ra{mine, inbox, s->mb_slot_floats, &((MailboxHdr *) s->mb_prev)->ack, s->d_in, (int) count};
    PeerRecvArgs rf = ra; rf.dst = s->d_final;
    PeerSendArgs sa{mine, (uint2 *)(s->mb_next + sizeof(MailboxHdr)), s->mb_slot_floats, s->d_out, (int) count};
    const int xfer_ctas = (int) std::min<size_t>(32, (count + 8191) / 8192);      // one CTA per 8 K elements, at most 32
    if (!sessions) { s->cur = session; s->cols = nullptr; }
    // fold the send into the slice's last matmul for plain single-token steps of quantised, head-size-128 slices
    const bool fold = s->use_fold && sends && !sessions && n_rows == 1 && s->D == 128 && s->wtype != kWT_F16 && s->use_ring &&
                      (!s->use_nq || wt_kquant(s->wtype)) &&
                      !s->skip_attention;
    const float * in = recv_in ? s->d_in : d_in;
    int rc = 0;
    auto body = [&]() -> int {
        int e;
        s->cur_class = 6;
        if (recv_in && (e = launch(s, k_peer_recv, dim3(xfer_ctas, 1, 1), dim3(1024, 1, 1), 0, ra))) return e;
        if (sends && !fold) { s->send_args = sa; s->send_pending = true; s->send_ctas = xfer_ctas; }
        s->fold_send = fold;
        e = enqueue_layers(s, in, n_rows, s->d_out);
        s->send_pending = false; s->fold_send = false;
        if (e) return e;
        s->cur_class = 6;
        if (recv_final && (e = launch(s, k_peer_recv, dim3(xfer_ctas, 1, 1), dim3(1024, 1, 1), 0, rf))) return e;
        return 0;
    };
    B200_CUDA(cudaEventRecord(s->ev0, s->stream));
    if (sessions) {
        if ((rc = begin_pass(s, sessions, counts, n_seq, n_rows))) return rc;
        rc = body();
        end_pass(s);
        if (rc) return rc;
        advance_pass(s, sessions, counts, n_seq);
    } else if (n_rows == 1 && s->use_graph && !s->profiling) {
        GraphKey key{in, nullptr, (ring & 3) | (fold ? 4 : 0) | (session << 3)};
        auto it = s->pp_graphs.find(key);
        if (it == s->pp_graphs.end()) {
            const int64_t before = s->launches;
            cudaGraph_t g = nullptr;
            B200_CUDA(cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeThreadLocal));
            rc = body();
            cudaError_t e = cudaStreamEndCapture(s->stream, &g);
            s->launches = before;
            if (rc) { if (g) cudaGraphDestroy(g); return rc; }
            if (e != cudaSuccess) return fail(B200_ECUDA, "pipeline graph capture failed: %s", cudaGetErrorString(e));
            cudaGraphExec_t ge = nullptr;
            e = cudaGraphInstantiate(&ge, g, 0);
            cudaGraphDestroy(g);
            if (e != cudaSuccess) return fail(B200_ECUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
            if (s->pp_graphs.size() >= 64) { for (auto & kv : s->pp_graphs) cudaGraphExecDestroy(kv.second); s->pp_graphs.clear(); }
            it = s->pp_graphs.emplace(key, ge).first;
        }
        B200_CUDA(cudaGraphLaunch(it->second, s->stream));
        s->launches += step_launches(s) + (recv_in ? 1 : 0) + (sends ? 1 : 0) + (recv_final ? 1 : 0);
        s->past[session] += 1;
    } else {
        s->cur = session; s->cols = nullptr;
        if ((rc = body())) return rc;
        s->past[session] += n_rows;
    }
    B200_CUDA(cudaEventRecord(s->ev1, s->stream));
    s->timed = true;
    return 0;
}

// recv <- rank-1, the slice's layers, send -> rank+1 (ring: the last rank hands its output back to rank 0).
// sessions == nullptr: n_rows tokens of session `session`; else a pass over the n_rows listed sessions, counts[k] tokens of
// sessions[k] (counts == nullptr: one each), and the hand-off is [sum of counts][n_embd].
static int pipeline_step_locked(b200_slice * s, const float * d_in, int n_rows, int ring, int session, const int * sessions,
                                const int * counts = nullptr) {
    NcclApi & n = nccl();
    B200_CUDA(cudaSetDevice(s->device));
    if (n_rows <= 0 || n_rows > s->n_ctx) return fail(B200_EINVAL, "n_tokens %d outside [1, n_ctx]", n_rows);
    const int n_seq = n_rows;
    const int r = s->pp_rank, W = s->pp_world;
    int rc;
    // validate the step BEFORE anything is posted: a rejected step must not leave the peer's send unmatched
    if (sessions) {
        if ((rc = check_pass(s, sessions, counts, n_seq, &n_rows))) return rc;
    } else {
        if (session < 0 || session >= s->n_sessions) return fail(B200_EINVAL, "session %d outside [0, %d)", session, s->n_sessions);
        if (s->past[session] + n_rows > s->n_ctx)
            return fail(B200_ECONTEXT, "context overflow: n_past %d + n_tokens %d > n_ctx %d", s->past[session], n_rows, s->n_ctx);
    }
    const size_t count = (size_t) n_rows * s->E;
    if (r == 0 && !d_in) return fail(B200_EINVAL, "rank 0 needs an input buffer");
    if (s->mb_on && W > 1) return pipeline_step_peer(s, d_in, n_rows, ring, session, sessions, counts, n_seq);
    const float * in = d_in;
    if (r > 0) {
        if ((rc = n.Recv(s->d_in, count, kNcclFloat32, r - 1, s->nccl_comm, s->stream))) return nccl_fail("ncclRecv", rc);
        in = s->d_in;
    }
    if (sessions) rc = pass_locked(s, sessions, counts, n_seq, in, s->d_out, false);
    else          rc = forward_locked(s, in, n_rows, s->d_out, false, session);
    if (rc) return rc;
    if (r < W - 1) {
        if ((rc = n.Send(s->d_out, count, kNcclFloat32, r + 1, s->nccl_comm, s->stream))) return nccl_fail("ncclSend", rc);
    } else if (ring && W > 1) {
        if ((rc = n.Send(s->d_out, count, kNcclFloat32, 0, s->nccl_comm, s->stream))) return nccl_fail("ncclSend", rc);
    }
    if (r == 0 && ring == 1 && W > 1) {
        // the last slice's output comes back to the first rank (where the client-side lm_head lives)
        if ((rc = n.Recv(s->d_final, count, kNcclFloat32, W - 1, s->nccl_comm, s->stream))) return nccl_fail("ncclRecv", rc);
    }
    s->launches += (r > 0) + (r < W - 1 || (ring && W > 1)) + (r == 0 && ring == 1 && W > 1);
    return 0;
}

int b200_pipeline_step(b200_slice_t * s, const float * d_in, int n_tokens, int ring) {
    if (!s || !s->nccl_comm) return fail(B200_EINVAL, "pipeline not initialised");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return pipeline_step_locked(s, d_in, n_tokens, ring, 0, nullptr);
}

int b200_pipeline_step_session(b200_slice_t * s, int session, const float * d_in, int n_tokens, int ring) {
    if (!s || !s->nccl_comm) return fail(B200_EINVAL, "pipeline not initialised");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return pipeline_step_locked(s, d_in, n_tokens, ring, session, nullptr);
}

int b200_pipeline_step_batch(b200_slice_t * s, const int * sessions, int n_seq, const float * d_in, int ring) {
    if (!s || !s->nccl_comm) return fail(B200_EINVAL, "pipeline not initialised");
    if (!sessions) return fail(B200_EINVAL, "null session list");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return pipeline_step_locked(s, d_in, n_seq, ring, 0, sessions);
}

int b200_pipeline_step_mixed(b200_slice_t * s, const int * sessions, const int * counts, int n_seq, const float * d_in, int ring) {
    if (!s || !s->nccl_comm) return fail(B200_EINVAL, "pipeline not initialised");
    if (!sessions || !counts) return fail(B200_EINVAL, "null session or count list");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    return pipeline_step_locked(s, d_in, n_seq, ring, 0, sessions, counts);
}

/* ---- peer-memory hand-off: mailboxes mapped across processes with cudaIpc --------------------------------------- */
int b200_pipeline_mailbox_export(b200_slice_t * s, void * handle64) {
    if (!s || !handle64) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    s->mb_slot_floats = (size_t) s->n_ctx * s->E;
    const size_t bytes = sizeof(MailboxHdr) + (size_t) kMbSlots * s->mb_slot_floats * 8;      // 8-byte {value, seq} elements
    if (!s->mb_block) {
        void * p = nullptr;
        B200_CUDA(cudaMalloc(&p, bytes));                 // a dedicated cudaMalloc block: IPC handles cover whole allocations
        s->allocs.push_back(p);
        s->mb_block = (uint8_t *) p;
    }
    // a fresh link: counters at zero, and sequence numbers start at 1, so a zeroed inbox holds no message
    B200_CUDA(cudaStreamSynchronize(s->stream));
    B200_CUDA(cudaMemset(s->mb_block, 0, bytes));
    s->use_fold = env_int("B200_PP_FOLD", 1) != 0;
    B200_CUDA(cudaDeviceSynchronize());
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    cudaIpcMemHandle_t h;
    B200_CUDA(cudaIpcGetMemHandle(&h, s->mb_block));
    memcpy(handle64, &h, 64);
    return 0;
}

int b200_pipeline_mailbox_connect(b200_slice_t * s, const void * handles, int nranks) {
    if (!s || !handles) return fail(B200_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (!s->mb_block) return fail(B200_EINVAL, "export this rank's mailbox first");
    if (nranks != s->pp_world || nranks < 2) return fail(B200_EINVAL, "mailbox_connect: %d handles for a pipeline of %d ranks", nranks, s->pp_world);
    if (env_int("B200_PP_PEER", 1) == 0) { s->mb_on = false; return 0; }       // keep the NCCL send/recv path (tested fallback)
    B200_CUDA(cudaSetDevice(s->device));
    const int next = (s->pp_rank + 1) % nranks, prev = (s->pp_rank + nranks - 1) % nranks;
    cudaIpcMemHandle_t hn, hp;
    memcpy(&hn, (const uint8_t *) handles + (size_t) next * 64, 64);
    memcpy(&hp, (const uint8_t *) handles + (size_t) prev * 64, 64);
    void * pn = nullptr, * pp = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&pn, hn, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(B200_ECUDA, "cudaIpcOpenMemHandle(next rank %d) failed: %s", next, cudaGetErrorString(e)); }
    if (prev == next) pp = pn;
    else {
        e = cudaIpcOpenMemHandle(&pp, hp, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { cudaGetLastError(); cudaIpcCloseMemHandle(pn); return fail(B200_ECUDA, "cudaIpcOpenMemHandle(previous rank %d) failed: %s", prev, cudaGetErrorString(e)); }
    }
    s->mb_next = (uint8_t *) pn; s->mb_prev = (uint8_t *) pp;
    s->mb_on = true;
    return 0;
}

/* Measurement aid: `iters` bare hand-offs of n_rows rows around the ring with NO layers in between (rank 0: send, recv;
 * others: recv, send), on the active transport; returns the device time per iteration in microseconds in *us_per_iter
 * (one iteration = `world` hops).  Every rank must call it. */
int b200_pipeline_pingpong(b200_slice_t * s, int n_rows, int iters, float * us_per_iter) {
    if (!s || !s->nccl_comm || !us_per_iter) return fail(B200_EINVAL, "pipeline not initialised");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    B200_CUDA(cudaSetDevice(s->device));
    const int r = s->pp_rank, W = s->pp_world;
    const size_t count = (size_t) n_rows * s->E;
    NcclApi & n = nccl();
    MailboxHdr * mine = (MailboxHdr *) s->mb_block;
    auto send = [&]() -> int {
        if (s->mb_on) {
            PeerSendArgs sa{mine, (uint2 *)(s->mb_next + sizeof(MailboxHdr)), s->mb_slot_floats, s->d_out, (int) count};
            return launch(s, k_peer_send, dim3((unsigned) std::min<size_t>(32, (count + 8191) / 8192), 1, 1), dim3(1024, 1, 1), 0, sa);
        }
        int rc = n.Send(s->d_out, count, kNcclFloat32, (r + 1) % W, s->nccl_comm, s->stream);
        return rc ? nccl_fail("ncclSend", rc) : 0;
    };
    auto recv = [&]() -> int {
        if (s->mb_on) {
            PeerRecvArgs ra{mine, (const uint2 *)(s->mb_block + sizeof(MailboxHdr)), s->mb_slot_floats, &((MailboxHdr *) s->mb_prev)->ack, s->d_in, (int) count};
            return launch(s, k_peer_recv, dim3((unsigned) std::min<size_t>(32, (count + 8191) / 8192), 1, 1), dim3(1024, 1, 1), 0, ra);
        }
        int rc = n.Recv(s->d_in, count, kNcclFloat32, (r + W - 1) % W, s->nccl_comm, s->stream);
        return rc ? nccl_fail("ncclRecv", rc) : 0;
    };
    cudaEvent_t e0, e1;
    B200_CUDA(cudaEventCreate(&e0)); B200_CUDA(cudaEventCreate(&e1));
    int rc = 0;
    for (int it = 0; it < iters + 8 && !rc; it++) {
        if (it == 8) cudaEventRecord(e0, s->stream);
        if (r == 0) { rc = send(); if (!rc) rc = recv(); }
        else        { rc = recv(); if (!rc) rc = send(); }
    }
    cudaEventRecord(e1, s->stream);
    cudaStreamSynchronize(s->stream);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    *us_per_iter = 1e3f * ms / (float) iters;
    return rc;
}

/* 1 when steps use the peer-memory mailboxes, 0 when they use ncclSend / ncclRecv. */
int b200_pipeline_transport(b200_slice_t * s) { return s && s->mb_on ? 1 : 0; }

/* Force the transport: 0 = NCCL (every rank must do the same, e.g. when ONE rank failed to map a neighbour),
 * 1 = peer mailboxes (only valid after a successful connect). */
int b200_pipeline_set_transport(b200_slice_t * s, int peer) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (peer && !(s->mb_next && s->mb_prev)) return fail(B200_EINVAL, "peer transport needs connected mailboxes");
    s->mb_on = peer != 0;
    return 0;
}

/* Non-zero if a mailbox poll timed out on this rank since the pipeline was connected (synchronises the stream). */
int b200_pipeline_error(b200_slice_t * s) {
    if (!s || !s->mb_block) return 0;
    cudaSetDevice(s->device);
    cudaStreamSynchronize(s->stream);
    int err = 0;
    cudaMemcpy(&err, s->mb_block + offsetof(MailboxHdr, err), 4, cudaMemcpyDeviceToHost);
    return err;
}

/* Rank 0: receive one final activation ([n_rows][n_embd]) that a step issued with ring = 2 left in flight, into d_dst
 * (NULL: the buffer b200_pipeline_result() returns).  Results arrive in the order the steps were issued.  Other ranks: no-op.
 * This is what keeps every slice busy in throughput mode: rank 0 issues steps for sessions k, k+1, ... back to back and
 * collects session k's result only when it needs it (rank r then works on session k while rank r+1 works on k-1). */
int b200_pipeline_collect(b200_slice_t * s, int n_rows, float * d_dst) {
    if (!s || !s->nccl_comm) return fail(B200_EINVAL, "pipeline not initialised");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (s->pp_rank != 0 || s->pp_world < 2) return 0;
    if (n_rows <= 0 || n_rows > s->n_ctx) return fail(B200_EINVAL, "n_rows %d outside [1, n_ctx]", n_rows);
    B200_CUDA(cudaSetDevice(s->device));
    float * dst = d_dst ? d_dst : s->d_final;
    const size_t count = (size_t) n_rows * s->E;
    if (s->mb_on) {
        PeerRecvArgs rf{(MailboxHdr *) s->mb_block, (const uint2 *)(s->mb_block + sizeof(MailboxHdr)), s->mb_slot_floats,
                        &((MailboxHdr *) s->mb_prev)->ack, dst, (int) count};
        s->cur_class = 6;
        int rc = launch(s, k_peer_recv, dim3((unsigned) std::min<size_t>(32, (count + 8191) / 8192), 1, 1), dim3(1024, 1, 1), 0, rf);
        if (rc) return rc;
    } else {
        NcclApi & n = nccl();
        int rc = n.Recv(dst, count, kNcclFloat32, s->pp_world - 1, s->nccl_comm, s->stream);
        if (rc) return nccl_fail("ncclRecv", rc);
        s->launches++;
    }
    return 0;
}

/* Device pointer of the pipeline's final activation on rank 0 (valid after a `ring` step), else dev_out. */
float * b200_pipeline_result(b200_slice_t * s) { return s ? (s->pp_world > 1 && s->pp_rank == 0 && s->d_final ? s->d_final : s->d_out) : nullptr; }

int b200_pipeline_destroy(b200_slice_t * s) {
    if (!s) return fail(B200_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(s->mu); B200_UNOWNED(s);
    if (s->nccl_comm) {
        cudaSetDevice(s->device);
        cudaStreamSynchronize(s->stream);
        NcclApi & n = nccl();
        if (n.CommDestroy) n.CommDestroy(s->nccl_comm);
        s->nccl_comm = nullptr; s->pp_world = 1; s->pp_rank = 0;
        for (auto & kv : s->pp_graphs) cudaGraphExecDestroy(kv.second);
        s->pp_graphs.clear();
        if (s->mb_next) cudaIpcCloseMemHandle(s->mb_next);
        if (s->mb_prev && s->mb_prev != s->mb_next) cudaIpcCloseMemHandle(s->mb_prev);
        s->mb_next = s->mb_prev = nullptr; s->mb_on = false;
    }
    return 0;
}

}  // extern "C"

// ============================================================================ client-side extra layers (N1)
// tok_embeddings lookup, final RMSNorm + lm_head, argmax, tokenizer -- resident, instead of the reference
// re-opening and re-reading the extra-layers file on every call (tensor_processor.cpp:1717-1908, 2033-2057,
// 2219-2235).  The lm_head is the same exact-mode weight matmul as the slice layers (RMSNorm prologue fused).
#include <queue>
#include <unordered_map>

struct b200_extra {
    b200_slice ctx;                       // device / stream / launch plumbing shared with the slice kernels
    int n_vocab = 0, E = 0, emb_type = 0, out_type = 0;
    uint8_t * emb_raw = nullptr;          // tok_embeddings as stored (row = token)
    float * norm_w = nullptr;
    PackedW out{}; uint16_t * out_f16 = nullptr;
    float * d_x = nullptr, * d_logits = nullptr; int32_t * d_tok = nullptr, * d_best = nullptr; int cap_tokens = 0;
    int32_t * d_ids = nullptr; int cap_ids = 0;    // generation: [n_steps][n_seq] ids; scoring: fed ids, then targets
    // sampling (k_sample_rows): per-row penalty bitmaps [rows][(n_vocab + 31) / 32], Philox keys, the first bad row
    uint32_t * d_pen = nullptr; uint64_t * d_seeds = nullptr; int * d_bad = nullptr; int cap_sample = 0;
    // scoring (b200_score): the embedded rows of one pass [rows][n_embd], and the NLL of every scored row
    float * d_sx = nullptr; int cap_sx = 0; double * d_nll = nullptr; int cap_nll = 0;
    // windowed perplexity (b200_perplexity_windows): every window's terms
    float * d_terms = nullptr; int cap_terms = 0;
    // log-probabilities (k_logprob_rows): lp [rows], top ids and their lp [rows][n_top]
    double * d_lp = nullptr; int cap_lp = 0; int32_t * d_topi = nullptr; int cap_topi = 0; double * d_topl = nullptr; int cap_topl = 0;
    // classifier-free guidance (k_cfg_rows): the guided rows [rows][n_vocab], kept apart so log-probabilities read raw rows
    float * d_cfg = nullptr; int cap_cfg = 0;
    std::vector<std::pair<std::string, float>> vocab;
    std::unordered_map<std::string, int> token_to_id;
    std::mutex mu;
};

namespace b200 {

__global__ void k_embed_rows(const uint8_t * emb, int type, int E, const int32_t * tok, int n_vocab, float * out) {
    const int n = blockIdx.y, t = tok[n];
    float * dst = out + (size_t) n * E;
    if (t < 0 || t >= n_vocab) { for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < E; i += gridDim.x * blockDim.x) dst[i] = 0.f; return; }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < E; i += gridDim.x * blockDim.x) {
        float v;
        if (wt_block_quant(type)) {
            v = deq32(emb + ((size_t) t * (E / 32) + i / 32) * wt_traits(type).block_bytes, type, i & 31);
        } else if (type == kWT_Q4_K) {
            v = dequant_q4k(emb + ((size_t) t * (E / 256) + i / 256) * 144, i & 255);
        } else if (type == kWT_F16) v = h2f(((const uint16_t *) emb)[(size_t) t * E + i]);
        else v = ((const float *) emb)[(size_t) t * E + i];
        dst[i] = v;
    }
}

static int extra_reserve(b200_extra * e, int n) {
    if (n <= e->cap_tokens) return 0;
    b200_slice * s = &e->ctx;
    // growth: release the old staging buffers first (they are tracked in `allocs` for unload)
    cudaStreamSynchronize(s->stream);
    for (void * old : {(void *) e->d_x, (void *) e->d_logits, (void *) e->d_tok, (void *) e->d_best, (void *) s->kq_aq, (void *) s->kq_ad}) {
        if (!old) continue;
        s->allocs.erase(std::remove(s->allocs.begin(), s->allocs.end(), old), s->allocs.end());
        cudaFree(old);
    }
    e->d_x = nullptr; e->d_logits = nullptr; e->d_tok = nullptr; e->d_best = nullptr; e->cap_tokens = 0;
    s->kq_aq = nullptr; s->kq_ad = nullptr;
    int rc;
    if ((rc = dev_alloc(s, &e->d_x, (size_t) n * e->E)) || (rc = dev_alloc(s, &e->d_logits, (size_t) n * e->n_vocab)) ||
        (rc = dev_alloc(s, &e->d_tok, (size_t) n)) || (rc = dev_alloc(s, &e->d_best, (size_t) 1))) return rc;
    if (e->out_type == kWT_Q6_K) {
        // the Q8_K rows of a Q6_K lm_head (quant_kq): its planes are laid out for ctx.n_ctx columns
        const int nbq = e->out.nbq;
        if ((rc = dev_alloc(s, &s->kq_aq, (size_t) n * nbq * (64 + 8))) || (rc = dev_alloc(s, &s->kq_ad, (size_t) n * kq_nbd(nbq)))) return rc;
        s->n_ctx = n;
    }
    e->cap_tokens = n;
    return 0;
}

static int extra_reserve_ids(b200_extra * e, int n) {
    if (n <= e->cap_ids) return 0;
    b200_slice * s = &e->ctx;
    cudaStreamSynchronize(s->stream);
    if (e->d_ids) {
        s->allocs.erase(std::remove(s->allocs.begin(), s->allocs.end(), (void *) e->d_ids), s->allocs.end());
        cudaFree(e->d_ids);
    }
    e->d_ids = nullptr; e->cap_ids = 0;
    if (int rc = dev_alloc(s, &e->d_ids, (size_t) n)) return rc;
    e->cap_ids = n;
    return 0;
}

static int extra_reserve_sample(b200_extra * e, int rows) {
    if (rows <= e->cap_sample) return 0;
    b200_slice * s = &e->ctx;
    cudaStreamSynchronize(s->stream);
    for (void * old : {(void *) e->d_pen, (void *) e->d_seeds, (void *) e->d_bad}) {
        if (!old) continue;
        s->allocs.erase(std::remove(s->allocs.begin(), s->allocs.end(), old), s->allocs.end());
        cudaFree(old);
    }
    e->d_pen = nullptr; e->d_seeds = nullptr; e->d_bad = nullptr; e->cap_sample = 0;
    int rc;
    if ((rc = dev_alloc(s, &e->d_pen, (size_t) rows * ((e->n_vocab + 31) / 32))) || (rc = dev_alloc(s, &e->d_seeds, (size_t) rows)) ||
        (rc = dev_alloc(s, &e->d_bad, (size_t) 1))) return rc;
    e->cap_sample = rows;
    return 0;
}

// Grows one of the extra layers' scratch buffers to n elements of T (its contents are not kept).
template <typename T> static int extra_regrow(b200_extra * e, T *& p, int & cap, size_t per, int n) {
    if (n <= cap) return 0;
    b200_slice * s = &e->ctx;
    cudaStreamSynchronize(s->stream);
    if (p) {
        s->allocs.erase(std::remove(s->allocs.begin(), s->allocs.end(), (void *) p), s->allocs.end());
        cudaFree(p);
    }
    p = nullptr; cap = 0;
    if (int rc = dev_alloc(s, &p, (size_t) n * per)) return rc;
    cap = n;
    return 0;
}

// sample_next_token (tensor_processor.cpp:1894-1908): best = -1e12, id = 0; `if (logit > best)` in index order, i.e. the
// FIRST maximum wins, NaNs never win, and a row that never exceeds -1e12 yields id 0.  One block over the row.
__global__ void __launch_bounds__(1024) k_argmax_first(const float * logits, int n, int32_t * out) {
    __shared__ float sv[32]; __shared__ int si[32];
    float bv = -(1000000000000.0f); int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float v = logits[i]; if (v > bv) { bv = v; bi = i; } }
    auto better = [](float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); };
    for (int o = 16; o > 0; o >>= 1) {
        const float v = __shfl_xor_sync(0xffffffffu, bv, o); const int i = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        bv = threadIdx.x < (blockDim.x >> 5) ? sv[threadIdx.x] : -(1000000000000.0f);
        bi = threadIdx.x < (blockDim.x >> 5) ? si[threadIdx.x] : 0x7fffffff;
        for (int o = 16; o > 0; o >>= 1) {
            const float v = __shfl_xor_sync(0xffffffffu, bv, o); const int i = __shfl_xor_sync(0xffffffffu, bi, o);
            if (better(v, i, bv, bi)) { bv = v; bi = i; }
        }
        if (threadIdx.x == 0) *out = bi == 0x7fffffff ? 0 : bi;
    }
}

// k_argmax_first's rule on one row of n logits, for a whole block: the id is valid in thread 0.
__device__ __forceinline__ int argmax_row(const float * logits, int n) {
    __shared__ float sv[32]; __shared__ int si[32];
    float bv = -(1000000000000.0f); int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float v = logits[i]; if (v > bv) { bv = v; bi = i; } }
    auto better = [](float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); };
    for (int o = 16; o > 0; o >>= 1) {
        const float v = __shfl_xor_sync(0xffffffffu, bv, o); const int i = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        bv = threadIdx.x < (blockDim.x >> 5) ? sv[threadIdx.x] : -(1000000000000.0f);
        bi = threadIdx.x < (blockDim.x >> 5) ? si[threadIdx.x] : 0x7fffffff;
        for (int o = 16; o > 0; o >>= 1) {
            const float v = __shfl_xor_sync(0xffffffffu, bv, o); const int i = __shfl_xor_sync(0xffffffffu, bi, o);
            if (better(v, i, bv, bi)) { bv = v; bi = i; }
        }
    }
    return bi == 0x7fffffff ? 0 : bi;
}

// The same rule for each of gridDim.x rows of [rows][n] logits, one block per row (k_argmax_first itself is kept apart so
// its code does not change).  Row k's id goes to tok[k], which the next step's embedding reads, and to ids[k].
__global__ void __launch_bounds__(1024) k_argmax_rows(const float * logits, int n, int32_t * tok, int32_t * ids) {
    const int k = blockIdx.x;
    const int best = argmax_row(logits + (size_t) k * n, n);
    if (threadIdx.x == 0) { tok[k] = best; ids[k] = best; }
}

// Word d (0-based) of numpy.random.Philox(key=seed): word d % 4 of Philox4x64-10 on counter (d / 4 + 1, 0, 0, 0) and
// key (seed, 0) -- numpy increments the counter before its first block.
__device__ __forceinline__ uint64_t philox_word(uint64_t seed, long long d) {
    uint64_t c0 = (uint64_t)(d >> 2) + 1, c1 = 0, c2 = 0, c3 = 0, k0 = seed, k1 = 0;
    for (int r = 0; r < 10; r++) {
        if (r) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
        const uint64_t hi0 = __umul64hi(0xD2E7470EE14C6C93ull, c0), lo0 = 0xD2E7470EE14C6C93ull * c0;
        const uint64_t hi1 = __umul64hi(0xCA5A826395121157ull, c2), lo1 = 0xCA5A826395121157ull * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    }
    const int w = (int)(d & 3);
    return w == 0 ? c0 : w == 1 ? c1 : w == 2 ? c2 : c3;
}

// Exclusive prefix sum over a warp in index order: lane l adds lanes 0 .. l-1 one at a time, so lane l + 1's result is
// lane l's result + v, bit for bit, and the prefixes never decrease.
__device__ __forceinline__ double warp_prefix_ordered(double v) {
    const int lane = threadIdx.x & 31;
    double p = 0.0;
    for (int j = 0; j < 31; j++) { const double w = __shfl_sync(0xffffffffu, v, j); if (j < lane) p = __dadd_rn(p, w); }
    return p;
}

// k_sample_rows: row k of [rows][n] logits is session k of the call.
struct SampleArgs {
    const float * logits; int n;
    double dt, dp;                   // the divisors: T + 1e-5, and rp * (T + 1e-5) for an id in prev
    const uint64_t * seeds; long long draw;   // row k takes draw `draw` of stream seeds[k]
    uint32_t * pen;                  // [rows][(n + 31) / 32]: bit i of row k = id i is in session k's prev
    int32_t * tok, * ids;            // the chosen id -> tok[k] (the next step's embedding reads it) and ids[k]
    int * bad; int bad_base;         // a row without a distribution: id -1, atomicMin(bad, bad_base + k)
    int top_k; double top_p;         // truncation; 0 = off
};

__device__ __forceinline__ double sample_weight(double dt, double dp, const float * x, const uint32_t * bits, int i, double m) {
    const double d = (bits[i >> 5] >> (i & 31)) & 1u ? dp : dt;
    return exp(__dsub_rn(__ddiv_rn((double) x[i], d), m));
}

// ---- sample_row's truncation stage (top-k / top-p): the kept ids are a prefix of the ranking (y descending, equal y lower
// id first), so one threshold per row describes them: id i is kept iff key_i > tau, or key_i == tau and i <= c.

__device__ __forceinline__ double sample_y(double dt, double dp, const float * x, const uint32_t * bits, int i) {
    const double d = (bits[i >> 5] >> (i & 31)) & 1u ? dp : dt;
    return __ddiv_rn((double) x[i], d);
}

// y as an unsigned integer in the order of y; -0 is folded onto +0, so equal y give equal keys.  (NaN rows never get here.)
__device__ __forceinline__ unsigned long long order_key(double y) {
    const unsigned long long b = (unsigned long long) __double_as_longlong(__dadd_rn(y, 0.0));
    return (b >> 63) ? ~b : b | 0x8000000000000000ull;
}

// sample_weight for a truncated row: the same arithmetic for a kept id, 0 for a dropped one.
__device__ __forceinline__ double kept_weight(double dt, double dp, const float * x, const uint32_t * bits, int i, double m,
                                              unsigned long long tau, int c) {
    const double y = sample_y(dt, dp, x, bits, i);
    const unsigned long long key = order_key(y);
    return key > tau || (key == tau && i <= c) ? exp(__dsub_rn(y, m)) : 0.0;
}

// Exclusive prefix of v over the block in thread order; *total = the block's sum.
__device__ __forceinline__ int block_scan_excl(int v, int * total) {
    __shared__ int s_w[33];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    int in = v;
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, in, o); if (lane >= o) in += u; }
    if (lane == 31) s_w[wid] = in;
    __syncthreads();
    if (wid == 0) {
        const int w = lane < nwarp ? s_w[lane] : 0;
        int wi = w;
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += u; }
        s_w[lane] = wi - w;
        if (lane == 31) s_w[32] = wi;
    }
    __syncthreads();
    const int r = s_w[wid] + in - v;
    *total = s_w[32];
    __syncthreads();                                    // s_w is free for the next call
    return r;
}

constexpr int kTruncCap = 1024;                         // candidates held on chip: one per thread of the 1024-thread block
struct TruncShared {
    unsigned long long key[kTruncCap], w[kTruncCap];    // the compacted candidates, in id order
    int id[kTruncCap];
    unsigned cnt[256]; unsigned long long mass[256];    // one level's histograms
    unsigned long long target, above_w, tau;            // block-uniform state of trunc_cut
    unsigned above_n, bin_n; int bin, ncand, c;
};

// One cut of a row's ranking -> (S.tau, S.c): the ranked id at which the running count reaches k (top-k), or at which the
// running weight within K first reaches ceil(p * S_K) (top-p; K = the ids kept by the cut (tk, ck) when kon).  Weights
// are fixed point, W_i = round(w_i * scale) with scale = 2^(63 - floor(log2 n)), so no sum can overflow 64 bits and any
// sum of them is exact whatever the order: counts and weights are shared-memory integer atomics.  The rounding error of a
// sum is at most n / (2 * scale), which relative to S_K >= 1 (the top id's weight is 1) is <= n * 2^(floor(log2 n) - 64).
// An MSB-first radix descent over the 64-bit keys, 8 bits a level: each level histograms the ids whose key matches the
// digits found so far, and warp 0 walks the bins from the top to the one where the running total reaches the target.
// Once the matching ids fit kTruncCap they are compacted on chip in id order (an ordered block scan) and the remaining
// levels read them there instead of the row.  After the last level the cut lies in a run of equal keys tau (equal y, so
// equal W): it takes the lowest j ids of the run, found with the ordered scan again.
__device__ __forceinline__ void trunc_cut(const float * x, int n, const uint32_t * bits, double dt, double dp, double m,
                                          double scale, bool by_mass, unsigned long long k, double p, bool kon,
                                          unsigned long long tk, int ck, TruncShared & S) {
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const int C = (n + blockDim.x - 1) / blockDim.x, i0 = min(n, t * C), i1 = min(n, i0 + C);
    if (t == 0) { S.target = k; S.above_w = 0; S.above_n = 0; }
    bool onchip = false;
    unsigned long long prefix = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        const int hs = shift + 8;                       // the bits above this digit must equal prefix's
        for (int b = t; b < 256; b += blockDim.x) { S.cnt[b] = 0; S.mass[b] = 0; }
        __syncthreads();
        if (onchip) {
            if (t < S.ncand) {
                const unsigned long long key = S.key[t];
                if (hs == 64 || (key >> hs) == (prefix >> hs)) {
                    const int dig = (int)(key >> shift) & 255;
                    atomicAdd(&S.cnt[dig], 1u);
                    if (by_mass) atomicAdd(&S.mass[dig], S.w[t]);
                }
            }
        } else {
            for (int i = i0; i < i1; i++) {
                const double y = sample_y(dt, dp, x, bits, i);
                const unsigned long long key = order_key(y);
                if ((hs < 64 && (key >> hs) != (prefix >> hs)) || (kon && (key < tk || (key == tk && i > ck)))) continue;
                const int dig = (int)(key >> shift) & 255;
                atomicAdd(&S.cnt[dig], 1u);
                if (by_mass) atomicAdd(&S.mass[dig], __double2ull_rn(__dmul_rn(exp(__dsub_rn(y, m)), scale)));
            }
        }
        __syncthreads();
        if (wid == 0) {                                 // lane l sums bins 255 - 8l .. 248 - 8l, then a scan from the top
            unsigned cn = 0; unsigned long long ms = 0;
            for (int j = 0; j < 8; j++) { cn += S.cnt[255 - 8 * lane - j]; ms += S.mass[255 - 8 * lane - j]; }
            unsigned ci = cn; unsigned long long mi = ms;
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned a = __shfl_up_sync(0xffffffffu, ci, o);
                const unsigned long long b = __shfl_up_sync(0xffffffffu, mi, o);
                if (lane >= o) { ci += a; mi += b; }
            }
            unsigned long long target = S.target;
            if (by_mass && shift == 56) {               // the first level holds all of K: S_K, and the target ceil(p S_K)
                const unsigned long long SK = __shfl_sync(0xffffffffu, mi, 31);
                target = min(max(__double2ull_ru(__dmul_rn(p, (double) SK)), 1ull), SK);
            }
            const unsigned long long aw = S.above_w; const unsigned an = S.above_n;
            const unsigned hit = __ballot_sync(0xffffffffu, by_mass ? aw + mi >= target : an + ci >= target);
            const int L = hit ? __ffs(hit) - 1 : 31;
            if (lane == L) {
                unsigned long long w = aw + mi - ms; unsigned c = an + ci - cn;
                int b = 255 - 8 * lane;
                for (int j = 0; j < 7; j++, b--) {
                    if (by_mass ? w + S.mass[b] >= target : c + S.cnt[b] >= target) break;
                    w += S.mass[b]; c += S.cnt[b];
                }
                S.bin = b; S.above_w = w; S.above_n = c; S.bin_n = S.cnt[b]; S.target = target;
            }
        }
        __syncthreads();
        prefix |= (unsigned long long) S.bin << shift;
        if (!onchip && shift > 0 && S.bin_n <= (unsigned) kTruncCap) {   // compact the candidates on chip, in id order
            int mine = 0;
            for (int i = i0; i < i1; i++) {
                const unsigned long long key = order_key(sample_y(dt, dp, x, bits, i));
                mine += (key >> shift) == (prefix >> shift) && !(kon && (key < tk || (key == tk && i > ck)));
            }
            int total;
            int at = block_scan_excl(mine, &total);
            for (int i = i0; i < i1 && mine; i++) {
                const double y = sample_y(dt, dp, x, bits, i);
                const unsigned long long key = order_key(y);
                if ((key >> shift) != (prefix >> shift) || (kon && (key < tk || (key == tk && i > ck)))) continue;
                S.key[at] = key; S.id[at] = i;
                S.w[at] = by_mass ? __double2ull_rn(__dmul_rn(exp(__dsub_rn(y, m)), scale)) : 0ull;
                at++; mine--;
            }
            if (t == 0) S.ncand = total;
            __syncthreads();
            onchip = true;
        }
    }
    // the run of keys == prefix holds the cut: the lowest j of its ids are kept
    unsigned long long j;
    if (by_mass) {
        const unsigned long long W = S.mass[S.bin] / S.bin_n, d = S.target - S.above_w;
        j = W ? d / W + (d % W != 0) : 1;
    } else {
        j = S.target - S.above_n;
    }
    if (t == 0) { S.tau = prefix; S.c = n - 1; }
    int mine = 0;
    if (onchip) mine = t < S.ncand && S.key[t] == prefix;
    else
        for (int i = i0; i < i1; i++) mine += order_key(sample_y(dt, dp, x, bits, i)) == prefix;
    int total;
    const int at = block_scan_excl(mine, &total);
    if ((unsigned long long) at < j && j <= (unsigned long long)(at + mine)) {
        if (onchip) S.c = S.id[t];
        else
            for (int i = i0, r = at; i < i1; i++)
                if (order_key(sample_y(dt, dp, x, bits, i)) == prefix && ++r == (int) j) { S.c = i; break; }
    }
    __syncthreads();
}

// The client's Sampler (cli_api/common.py:64-86) on one row x of n logits, for a whole block: divisors dt / dp, penalty
// bitmap bits, u = draw `draw` of Philox stream `seed`.  The id is valid in thread 0; -1 when the row has no
// distribution.  Thread t owns the contiguous chunk [t*C, t*C + C) of the row.
//   1. max y: the divisor takes two values and a correctly rounded division is monotone, so max y is the larger of
//      (max x over ids outside prev) / dt and (max x over ids in prev) / dp.  A NaN, or a max that is not finite, is a
//      row numpy rejects.
//   2. e_i = exp(y_i - max y) in float64; each thread sums its chunk in order; the chunk offsets O_t are an ordered scan
//      (warp_prefix_ordered within and across warps), so they never decrease and O_t + total_t is O_{t+1} exactly.
//   3. The thread whose [O_t, O_{t+1}) holds u*S (S the total; the last chunk with weight when u*S rounds to S) claims
//      the draw; warp 0 re-walks that chunk in order from O_t and picks the first id whose running sum passes u*S,
//      falling back to the chunk's last id of positive weight.  An id of weight 0 never moves the sum, so it is never
//      picked.  The row's logits are read from L2 in each pass.
// With truncation on (0 < top_k < n, or 0 < top_p < 1: a block-uniform branch), a stage between 1 and 2 finds the row's
// threshold (tau, c) with trunc_cut -- top-k first, then top-p within K -- and steps 2 and 3 use weight 0 for every id
// it drops, in the same chunks and order.  So dropping ids whose weight is already 0 changes no bit.  With truncation
// off, steps 2 and 3 are the untruncated arithmetic.
__device__ __forceinline__ int sample_row(const float * x, int n, const uint32_t * bits, double dt, double dp, uint64_t seed,
                                          long long draw, int top_k, double top_p) {
    __shared__ float smf[32], smp[32];
    __shared__ double swt[32], swo[32], s_m, s_u, s_total, s_target, s_o;
    __shared__ int s_chunk;
    __shared__ TruncShared s_trunc;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5, nwarp = blockDim.x >> 5;
    const int C = (n + blockDim.x - 1) / blockDim.x, i0 = min(n, t * C), i1 = min(n, i0 + C);
    float mf = -INFINITY, mp = -INFINITY; bool nan = false;
    for (int i = i0; i < i1; i++) {
        const float v = x[i];
        nan |= v != v;
        if ((bits[i >> 5] >> (i & 31)) & 1u) mp = fmaxf(mp, v); else mf = fmaxf(mf, v);
    }
    for (int o = 16; o > 0; o >>= 1) {
        mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o)); mp = fmaxf(mp, __shfl_xor_sync(0xffffffffu, mp, o));
    }
    if (lane == 0) { smf[wid] = mf; smp[wid] = mp; }
    if (t == 0) s_chunk = 0x7fffffff;
    const bool any_nan = __syncthreads_or(nan);
    if (wid == 0) {
        mf = lane < nwarp ? smf[lane] : -INFINITY; mp = lane < nwarp ? smp[lane] : -INFINITY;
        for (int o = 16; o > 0; o >>= 1) {
            mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o)); mp = fmaxf(mp, __shfl_xor_sync(0xffffffffu, mp, o));
        }
        if (lane == 0) {
            s_m = fmax(__ddiv_rn((double) mf, dt), __ddiv_rn((double) mp, dp));
            s_u = (double)(philox_word(seed, draw) >> 11) * 0x1.0p-53;
        }
    }
    __syncthreads();
    const double m = s_m;
    if (any_nan || !isfinite(m)) return -1;
    const bool trunc = (top_k > 0 && top_k < n) || (top_p > 0.0 && top_p < 1.0);
    unsigned long long tau = 0; int cut = 0;
    if (trunc) {
        const double scale = ldexp(1.0, 63 - (31 - __clz(n)));
        bool kon = false;
        if (top_k > 0 && top_k < n) {
            trunc_cut(x, n, bits, dt, dp, m, scale, false, (unsigned long long) top_k, 0.0, false, 0, 0, s_trunc);
            kon = true; tau = s_trunc.tau; cut = s_trunc.c;
        }
        if (top_p > 0.0 && top_p < 1.0) {
            trunc_cut(x, n, bits, dt, dp, m, scale, true, 0, top_p, kon, tau, cut, s_trunc);
            tau = s_trunc.tau; cut = s_trunc.c;
        }
    }
    double tot = 0.0;
    if (trunc) for (int i = i0; i < i1; i++) tot = __dadd_rn(tot, kept_weight(dt, dp, x, bits, i, m, tau, cut));
    else       for (int i = i0; i < i1; i++) tot = __dadd_rn(tot, sample_weight(dt, dp, x, bits, i, m));
    const double P = warp_prefix_ordered(tot), Pin = __dadd_rn(P, tot);
    if (lane == 31) swt[wid] = Pin;
    __syncthreads();
    if (wid == 0) {
        const double v = lane < nwarp ? swt[lane] : 0.0, W = warp_prefix_ordered(v);
        swo[lane] = W;
        if (lane == 31) { const double S = __dadd_rn(W, v); s_target = __dmul_rn(s_u, S); s_total = S; }
    }
    __syncthreads();
    const double S = s_total, target = s_target;
    const double O = __dadd_rn(swo[wid], P), Oend = __dadd_rn(swo[wid], Pin);
    if (tot > 0.0 && O <= target && (target < Oend || Oend == S)) atomicMin(&s_chunk, t);
    __syncthreads();
    if (t == s_chunk) s_o = O;
    __syncthreads();
    if (wid != 0) return -1;
    const int j0 = min(n, s_chunk * C), j1 = min(n, j0 + C);
    double r = s_o; int id = -1, last = -1;
    for (int b = j0; b < j1 && id < 0; b += 32) {
        const int i = b + lane;
        const double e = i >= j1 ? 0.0 : trunc ? kept_weight(dt, dp, x, bits, i, m, tau, cut) : sample_weight(dt, dp, x, bits, i, m);
        double q = r;                                  // r + e_b + ... + e_i, added in index order
        for (int j = 0; j < 32; j++) { const double w = __shfl_sync(0xffffffffu, e, j); if (j <= lane) q = __dadd_rn(q, w); }
        const unsigned hit = __ballot_sync(0xffffffffu, i < j1 && q > target);
        const unsigned pos = __ballot_sync(0xffffffffu, i < j1 && e > 0.0);
        if (hit) id = b + __ffs(hit) - 1;
        if (pos) last = b + 31 - __clz(pos);
        r = __shfl_sync(0xffffffffu, q, 31);
    }
    return id < 0 ? last : id;
}

// k_sample_rows: sample_row on each of gridDim.x rows, one block per row; row k is session k of the call.
__global__ void __launch_bounds__(1024) k_sample_rows(SampleArgs a) {
    const int k = blockIdx.x;
    uint32_t * bits = a.pen + (size_t) k * ((a.n + 31) >> 5);
    const int id = sample_row(a.logits + (size_t) k * a.n, a.n, bits, a.dt, a.dp, a.seeds[k], a.draw, a.top_k, a.top_p);
    if (threadIdx.x != 0) return;
    a.tok[k] = id; a.ids[k] = id;
    if (id < 0) atomicMin(a.bad, a.bad_base + k);
    else bits[id >> 5] |= 1u << (id & 31);
}

// ---- generation streams (b200_stream_*): the sampler's state lives in per-session slots, and a step's rows name their slot
struct StreamSlot { uint64_t seed; double dt, dp; int sampled, top_k; double top_p; };   // device table, one per session
struct StreamRow { long long draw; int slot, gather, n_top, gather2; };   // per step, in mapped pinned memory: draw index,
                                                                    // slot, the session's last row in the pass, its top-n
                                                                    // (-1: no log-probabilities), and its guidance
                                                                    // session's last row (-1: unguided)

// A step's token rows: row r is the prompt id spec[r] when spec[r] >= 0, else the last id slot ~spec[r] drew.  spec lies in
// mapped pinned memory.
__global__ void k_stream_tokens(const int32_t * spec, const int32_t * last, int n, int32_t * tok) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        const int32_t v = spec[r];
        tok[r] = v >= 0 ? v : last[~v];
    }
}

// A stream step with no draw (only non-final prompt chunks) publishes its completion here instead: cell 0 of its publish
// ring, which the host set to INT32_MIN, so the region is not reused before the step's k_stream_tokens has read it.
__global__ void k_stream_mark(int32_t * cell) { *(volatile int32_t *) cell = 0; }

// Row k of out is row rows[k].gather of x (rows[k].gather2 when second): each session's last row of a mixed pass, or its
// guidance session's, packed for the lm_head.
__global__ void k_gather_rows(const float * x, const StreamRow * rows, int E, float * out, bool second = false) {
    __shared__ int g;
    if (threadIdx.x == 0) g = second ? rows[blockIdx.y].gather2 : rows[blockIdx.y].gather;
    __syncthreads();
    const float * src = x + (size_t) g * E;
    float * dst = out + (size_t) blockIdx.y * E;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < E; i += gridDim.x * blockDim.x) dst[i] = src[i];
}

// One id for each of gridDim.x rows of [rows][n] logits, row k for slot rows[k].slot: the argmax rule on the raw logits for
// a greedy slot (argmax_row), the Sampler with the slot's divisors, key and the row's draw index for a sampled one
// (sample_row, which then marks the id in the slot's penalty bitmap).  The id becomes the slot's last id, which the next
// step's k_stream_tokens reads, and is stored into cell k of the step's publish ring in mapped pinned memory: the host
// sets every cell to INT32_MIN before it enqueues the step, so each cell carries its own readiness.  A row that asked for
// log-probabilities is published by k_stream_logprobs instead, after its record.  Guided rows (logits: k_cfg_rows' rows)
// take a greedy slot's id from pick[k], k_cfg_rows' max_element pick, instead of the argmax.
__global__ void __launch_bounds__(1024) k_stream_draw(const float * logits, int n, const StreamRow * rows,
                                                      const StreamSlot * slots, uint32_t * pen, int32_t * last, int32_t * ring,
                                                      const int32_t * pick = nullptr) {
    __shared__ StreamRow s_row;
    const int k = blockIdx.x;
    if (threadIdx.x == 0) s_row = rows[k];
    __syncthreads();
    const int slot = s_row.slot;
    const StreamSlot sl = slots[slot];
    const float * x = logits + (size_t) k * n;
    uint32_t * bits = pen + (size_t) slot * ((n + 31) >> 5);
    const int id = sl.sampled ? sample_row(x, n, bits, sl.dt, sl.dp, sl.seed, s_row.draw, sl.top_k, sl.top_p)
                              : pick ? pick[k] : argmax_row(x, n);
    if (threadIdx.x != 0) return;
    if (sl.sampled && id >= 0) bits[id >> 5] |= 1u << (id & 31);
    last[slot] = id;
    if (s_row.n_top < 0) *(volatile int32_t *)(ring + k) = id;
}

// The client's perplexity term (cli_api/common.py:129-139) for each of gridDim.x rows of [rows][n] logits, one block per
// row: nll[k] = -log(e_t / S) with t = tgt[k], e_i = exp((double) x_i - m), m = max x and S = sum e_i, all in float64.
// Thread t sums its contiguous chunk [t*C, t*C + C) in order and the chunk totals combine in index order
// (warp_prefix_ordered within and across warps, as in k_sample_rows), so a row's value depends only on its logits and its
// target.  Non-finite rows follow numpy: a NaN or +inf logit, or a row that is all -inf, gives NaN; a target whose e_t
// underflows gives +inf.
// The softmax normaliser of that term for one row x of n logits, for a whole block: m and S, valid in every thread.  Returns
// false (block-uniform) when the row has no distribution.  k_nll_rows and k_logprob_rows both take m and S from here, so a
// log-probability is exactly the negated NLL of the same row and id.
__device__ __forceinline__ bool row_softmax(const float * x, int n, double * m_out, double * s_out) {
    __shared__ float smx[32];
    __shared__ double swt[32], s_S;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5, nwarp = blockDim.x >> 5;
    const int C = (n + blockDim.x - 1) / blockDim.x, i0 = min(n, t * C), i1 = min(n, i0 + C);
    float mx = -INFINITY; bool bad = false;
    for (int i = i0; i < i1; i++) { const float v = x[i]; bad |= v != v || v == INFINITY; mx = fmaxf(mx, v); }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) smx[wid] = mx;
    const bool any_bad = __syncthreads_or(bad);
    mx = lane < nwarp ? smx[lane] : -INFINITY;          // every warp reduces the warp maxima: m is block-uniform
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (any_bad || mx == -INFINITY) return false;
    const double m = (double) mx;
    double tot = 0.0;
#pragma unroll 1                                         // unrolled, the float64 exp spills at 32 registers (2 CTAs / SM)
    for (int i = i0; i < i1; i++) tot = __dadd_rn(tot, exp(__dsub_rn((double) x[i], m)));
    const double P = warp_prefix_ordered(tot);
    if (lane == 31) swt[wid] = __dadd_rn(P, tot);
    __syncthreads();
    if (wid == 0) {
        const double v = lane < nwarp ? swt[lane] : 0.0, W = warp_prefix_ordered(v);
        if (lane == 31) s_S = __dadd_rn(W, v);
    }
    __syncthreads();
    *m_out = m; *s_out = s_S;
    return true;
}

// log(e_t / S) for a logit x_t of a row with normaliser (m, S): -inf when e_t underflows.
__device__ __forceinline__ double row_logp(float xt, double m, double S) {
    return log(__ddiv_rn(exp(__dsub_rn((double) xt, m)), S));
}

__global__ void __launch_bounds__(1024) k_nll_rows(const float * logits, int n, const int32_t * tgt, double * nll) {
    const int k = blockIdx.x;
    const float * x = logits + (size_t) k * n;
    double m, S;
    const bool ok = row_softmax(x, n, &m, &S);
    if (threadIdx.x == 0) nll[k] = ok ? -row_logp(x[tgt[k]], m, S) : __longlong_as_double(0x7ff8000000000000ll);
}

// ---- llama.cpp's perplexity term (b200_perplexity_windows, b200_extra_ppl_terms): perplexity.cpp:12-26 and 103-113.
// For a row x of n logits and target t: m = max x, e_i = expf(x_i - m) with the subtraction in float, S = the e_i summed
// in double strictly in index order 0 .. n-1, prob = (float)(e_t / S), term = -logf(prob) (std::log of a float is the
// float overload).  expf / logf here are the double functions rounded to float; perplexity.cpp calls glibc's, which are
// not correctly rounded near float midpoints, so that is the one place the two can give different bits.  A row with a
// NaN or +inf logit, or all -inf, gives NaN (as k_nll_rows); a prob that underflows to 0 gives +inf.
// The ordered sum is a dependent chain of n double additions per row, so a block takes kPplRows rows at once: warp w < 8
// finds row w's max, then warps 1.. compute the e_i of a tile of every row into shared memory while lane r of warp 0 adds
// the previous tile's row-r values to its one accumulator (double-buffered; rows padded a float so the eight summing
// lanes read eight banks).
constexpr int kPplRows = 8, kPplTile = 512, kPplThreads = 256;

__device__ __forceinline__ float ppl_expf(float v) { return __double2float_rn(exp((double) v)); }

__global__ void __launch_bounds__(kPplThreads) k_ppl_rows(const float * logits, int n, int n_rows, const int32_t * tgt,
                                                          float * term) {
    __shared__ float s_e[2][kPplRows][kPplTile + 1];
    __shared__ float s_m[kPplRows];
    __shared__ int s_ok[kPplRows];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const int r0 = blockIdx.x * kPplRows, nr = min(kPplRows, n_rows - r0);
    if (wid < nr) {
        const float * x = logits + (size_t)(r0 + wid) * n;
        float mx = -INFINITY; bool bad = false;
        for (int i = lane; i < n; i += 32) { const float v = x[i]; bad |= v != v || v == INFINITY; mx = fmaxf(mx, v); }
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        bad = __any_sync(0xffffffffu, bad);
        if (lane == 0) { s_m[wid] = mx; s_ok[wid] = !bad && mx != -INFINITY; }
    }
    __syncthreads();
    const int n_tiles = (n + kPplTile - 1) / kPplTile;
    auto produce = [&](int tile) {                        // warps 1..: e_i of columns [tile * kPplTile, +kPplTile)
        const int c0 = tile * kPplTile, cn = min(kPplTile, n - c0);
        float (*dst)[kPplTile + 1] = s_e[tile & 1];
        for (int idx = t - 32; idx < nr * kPplTile; idx += kPplThreads - 32) {
            const int r = idx / kPplTile, c = idx % kPplTile;
            if (c < cn) dst[r][c] = ppl_expf(__fsub_rn(logits[(size_t)(r0 + r) * n + c0 + c], s_m[r]));
        }
    };
    if (wid > 0) produce(0);
    __syncthreads();
    double S = 0.0;
    for (int k = 0; k < n_tiles; k++) {
        if (wid > 0) {
            if (k + 1 < n_tiles) produce(k + 1);
        } else if (t < nr) {
            const float * e = s_e[k & 1][t];
            const int cn = min(kPplTile, n - k * kPplTile);
#pragma unroll 8
            for (int c = 0; c < cn; c++) S = __dadd_rn(S, (double) e[c]);
        }
        __syncthreads();
    }
    if (t < nr) {
        const int r = r0 + t;
        float out = __int_as_float(0x7fc00000);
        if (s_ok[t]) {
            const float et = ppl_expf(__fsub_rn(logits[(size_t) r * n + tgt[r]], s_m[t]));
            const float prob = __double2float_rn(__ddiv_rn((double) et, S));
            out = -__double2float_rn(log((double) prob));
        }
        term[r] = out;
    }
}

// ---- llama.cpp's classifier-free guidance (b200_generate_cfg, b200_extra_cfg): llama_sample_classifier_free_guidance
// (llama.cpp:2170-2225) on a pair of rows, b the session's logits and g its guidance session's:
//   log_softmax(v): m = *max_element(v) (v_0 when v_0 is NaN, else the largest non-NaN v_i), p_i = expf(v_i - m), S = the
//     p_i summed in FLOAT strictly in index order, v_i = logf(p_i / S);
//   lb = log_softmax(b), lg = log_softmax(g), mix_i = fmaf(scale, lb_i - lg_i, lg_i), lg2 = log_softmax(mix),
//   out_i = fmaf(sf, lg2_i, (1 - sf) * lb_i)
// with the two FMAs the reference build contracts (vfmadd132ss, vfmadd231ss) and nothing else fused.  expf / logf are the
// double functions rounded to float (ppl_expf, cfg_logf), so glibc's, which are not correctly rounded everywhere, are the
// one place the reference can give other bits.  The float sums are dependent chains of n additions, so k_ppl_rows' shape:
// producer warps fill tiles of p_i into shared memory while lanes 0 and 1 of warp 0 add b's and g's in order, then the mix
// chain on lane 0.  The logs are recomputed from the inputs where needed (no n-float scratch besides the output row, which
// holds mix until the last phase overwrites it).
// pick[k] is max_element(out) (llama_sample_token_greedy: out_0 when it is NaN, else the first largest non-NaN value), or
// -1 when b or g has no distribution (a NaN or +inf, or all -inf); then, when bad is given, atomicMin(bad, bad_base + k).
constexpr int kCfgTile = 512, kCfgThreads = 256;

__device__ __forceinline__ float cfg_logf(float v) { return __double2float_rn(log((double) v)); }

struct CfgArgs {
    const float * base, * guid;     // row k of each: [rows][n]
    int n;
    float scale, sf;
    float * out;                    // [rows][n]
    int32_t * pick, * pick2;        // [rows], either may be NULL (generation: the next step's token and the call's ids)
    int * bad; int bad_base;        // may be NULL
};

// max_element's value over x[0, n) (NaN when x_0 is NaN) and whether x has a distribution, for a whole block.
__device__ __forceinline__ float cfg_row_max(const float * x, int n, bool * ok) {
    __shared__ float s_mx[32]; __shared__ int s_bad[32];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5, nwarp = blockDim.x >> 5;
    float mx = -INFINITY; bool bad = false;
    for (int i = t; i < n; i += blockDim.x) { const float v = x[i]; bad |= v != v || v == INFINITY; mx = fmaxf(mx, v); }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    bad = __any_sync(0xffffffffu, bad);
    __syncthreads();                                     // the previous call's readers are done with s_mx
    if (lane == 0) { s_mx[wid] = mx; s_bad[wid] = bad; }
    __syncthreads();
    mx = lane < nwarp ? s_mx[lane] : -INFINITY;
    bad = lane < nwarp ? s_bad[lane] : false;
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    bad = __any_sync(0xffffffffu, bad);
    *ok = !bad && mx != -INFINITY;
    const float x0 = x[0];
    return x0 != x0 ? x0 : mx;
}

// The in-order float sums of expf(x_r[i] - m[r]) for nr (1 or 2) rows, lane r of warp 0 holding row r's chain; every
// thread gets them in S[0 .. nr).
__device__ __forceinline__ void cfg_chains(const float * const * x, const float * m, int nr, int n, float * S) {
    __shared__ float s_e[2][2][kCfgTile + 1];
    __shared__ float s_S[2];
    const int t = threadIdx.x, wid = t >> 5;
    const int n_tiles = (n + kCfgTile - 1) / kCfgTile;
    auto produce = [&](int tile) {
        const int c0 = tile * kCfgTile, cn = min(kCfgTile, n - c0);
        for (int idx = t - 32; idx < nr * kCfgTile; idx += kCfgThreads - 32) {
            const int r = idx / kCfgTile, c = idx % kCfgTile;
            if (c < cn) s_e[tile & 1][r][c] = ppl_expf(__fsub_rn(x[r][c0 + c], m[r]));
        }
    };
    if (wid > 0) produce(0);
    __syncthreads();
    float acc = 0.f;
    for (int k = 0; k < n_tiles; k++) {
        if (wid > 0) {
            if (k + 1 < n_tiles) produce(k + 1);
        } else if (t < nr) {
            const float * e = s_e[k & 1][t];
            const int cn = min(kCfgTile, n - k * kCfgTile);
#pragma unroll 8
            for (int c = 0; c < cn; c++) acc = __fadd_rn(acc, e[c]);
        }
        __syncthreads();
    }
    if (t < nr) s_S[t] = acc;
    __syncthreads();
    for (int r = 0; r < nr; r++) S[r] = s_S[r];
}

__global__ void __launch_bounds__(kCfgThreads) k_cfg_rows(CfgArgs a) {
    __shared__ float s_v[32]; __shared__ int s_i[32];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5, nwarp = blockDim.x >> 5, n = a.n;
    const size_t k = blockIdx.x;
    const float * b = a.base + k * n, * g = a.guid + k * n;
    float * out = a.out + k * n;
    bool ok_b, ok_g;
    float m[2];
    m[0] = cfg_row_max(b, n, &ok_b);
    m[1] = cfg_row_max(g, n, &ok_g);
    const float * rows[2] = {b, g};
    float S[2];
    cfg_chains(rows, m, 2, n, S);
    auto lb_at = [&](int i) { return cfg_logf(__fdiv_rn(ppl_expf(__fsub_rn(b[i], m[0])), S[0])); };
    for (int i = t; i < n; i += blockDim.x) {
        const float lb = lb_at(i), lg = cfg_logf(__fdiv_rn(ppl_expf(__fsub_rn(g[i], m[1])), S[1]));
        out[i] = __fmaf_rn(a.scale, __fsub_rn(lb, lg), lg);
    }
    __syncthreads();                                     // out (the mix row) is visible to the whole block
    bool ok_mix;                                         // unused: a mix row without a distribution is NaN by arithmetic
    float m2[1] = {cfg_row_max(out, n, &ok_mix)};
    const float * mrow[1] = {out};
    float S2[1];
    cfg_chains(mrow, m2, 1, n, S2);
    const float one_minus = __fsub_rn(1.f, a.sf);
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int i = t; i < n; i += blockDim.x) {
        const float lg2 = cfg_logf(__fdiv_rn(ppl_expf(__fsub_rn(out[i], m2[0])), S2[0]));
        const float v = __fmaf_rn(a.sf, lg2, __fmul_rn(one_minus, lb_at(i)));
        out[i] = v;
        if (v > bv) { bv = v; bi = i; }                  // NaN never wins; ascending i keeps the first of equals
    }
    auto better = [](float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); };
    for (int o = 16; o > 0; o >>= 1) {
        const float v = __shfl_xor_sync(0xffffffffu, bv, o); const int i = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
    if (lane == 0) { s_v[wid] = bv; s_i[wid] = bi; }
    __syncthreads();
    if (t != 0) return;
    bv = s_v[0]; bi = s_i[0];
    for (int w = 1; w < nwarp; w++) if (better(s_v[w], s_i[w], bv, bi)) { bv = s_v[w]; bi = s_i[w]; }
    const float o0 = out[0];
    const int id = !(ok_b && ok_g) ? -1 : (o0 != o0 || bi == 0x7fffffff) ? 0 : bi;
    if (a.pick) a.pick[k] = id;
    if (a.pick2) a.pick2[k] = id;
    if (id < 0 && a.bad) atomicMin(a.bad, a.bad_base + (int) k);
}

// ---- log-probabilities of drawn ids (b200_generate_lp, b200_stream_read_lp, b200_extra_logprobs): the raw distribution
// softmax(x) of row_softmax, whatever the sampler's settings, and the n_top ids of largest x beside the drawn one.
constexpr int kMaxTop = 20;

// (a, ia) ranks before (b, ib): larger x first, equal x lower id first.  (Rows with a NaN never get here.)
__device__ __forceinline__ bool ranks_before(float a, int ia, float b, int ib) { return a > b || (a == b && ia < ib); }

// The best-ranked id of x[i0, i1) that ranks strictly after (pv, pi); (-inf, INT_MAX) when there is none.
__device__ __forceinline__ void chunk_next(const float * x, int i0, int i1, float pv, int pi, float & bv, int & bi) {
    bv = -INFINITY; bi = 0x7fffffff;
    for (int i = i0; i < i1; i++) {
        const float v = x[i];
        if (ranks_before(pv, pi, v, i) && ranks_before(v, i, bv, bi)) { bv = v; bi = i; }
    }
}

__device__ __forceinline__ void warp_best(float & v, int & i) {
    for (int o = 16; o > 0; o >>= 1) {
        const float w = __shfl_xor_sync(0xffffffffu, v, o); const int j = __shfl_xor_sync(0xffffffffu, i, o);
        if (ranks_before(w, j, v, i)) { v = w; i = j; }
    }
}

// lp = log p(id) and the n_top best-ranked ids with theirs, for one row of n logits, for a whole block.  A row without a
// distribution (row_softmax) gives NaN and ids -1; so does lp of an id < 0.  The top-n: each thread keeps the best-ranked
// id of its chunk not picked yet; a round reduces those over the block to the next pick, and the thread that owned it
// rescans its own chunk.  So a round reads C logits, and the rank order is total, so the picks are exact on ties.
__device__ __forceinline__ void logprob_row(const float * x, int n, int id, int n_top, double * lp, int32_t * top_ids,
                                            double * top_lp) {
    __shared__ float s_v[32]; __shared__ int s_i[32], s_pick[kMaxTop];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5, nwarp = blockDim.x >> 5;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double m, S;
    if (!row_softmax(x, n, &m, &S)) {
        if (t == 0) *lp = nan;
        if (t < n_top) { top_ids[t] = -1; top_lp[t] = nan; }
        return;
    }
    if (t == 0) *lp = id >= 0 ? row_logp(x[id], m, S) : nan;
    if (n_top == 0) return;
    const int C = (n + blockDim.x - 1) / blockDim.x, i0 = min(n, t * C), i1 = min(n, i0 + C);
    float bv; int bi;
    chunk_next(x, i0, i1, INFINITY, -1, bv, bi);
    for (int r = 0; r < n_top; r++) {
        float v = bv; int i = bi;
        warp_best(v, i);
        if (lane == 0) { s_v[wid] = v; s_i[wid] = i; }
        __syncthreads();
        v = lane < nwarp ? s_v[lane] : -INFINITY; i = lane < nwarp ? s_i[lane] : 0x7fffffff;
        warp_best(v, i);                                // every warp reduces the warp bests: the pick is block-uniform
        if (t == 0) s_pick[r] = i;
        if (i >= i0 && i < i1) chunk_next(x, i0, i1, v, i, bv, bi);
        __syncthreads();
    }
    if (t < n_top) { const int j = s_pick[t]; top_ids[t] = j; top_lp[t] = row_logp(x[j], m, S); }
}

// logprob_row on each of gridDim.x rows of [rows][n] logits: row k's id is ids[k], its outputs lp[k] and
// top_ids / top_lp [k][n_top].
__global__ void __launch_bounds__(1024) k_logprob_rows(const float * logits, int n, const int32_t * ids, int n_top, double * lp,
                                                       int32_t * top_ids, double * top_lp) {
    const size_t k = blockIdx.x;
    logprob_row(logits + k * n, n, ids[k], n_top, lp + k, top_ids + k * n_top, top_lp + k * n_top);
}

// A row's log-probability record in a stream's mapped logprob ring, one cell per publish-ring cell.
struct LpRecord { double lp; int32_t top_ids[kMaxTop]; double top_lp[kMaxTop]; };
static_assert(sizeof(LpRecord) == 8 + kMaxTop * 12, "LpRecord layout");

// The records of a step's rows that asked for log-probabilities (the others return at once), launched after k_stream_draw:
// row k's id is its slot's last id.  Every thread's stores into the mapped record reach the system before the id enters
// publish cell k, so a host that sees the id also sees the record.
__global__ void __launch_bounds__(1024) k_stream_logprobs(const float * logits, int n, const StreamRow * rows,
                                                          const int32_t * last, int32_t * ring, LpRecord * rec) {
    __shared__ StreamRow s_row;
    const int k = blockIdx.x;
    if (threadIdx.x == 0) s_row = rows[k];
    __syncthreads();
    if (s_row.n_top < 0) return;
    const int id = last[s_row.slot];
    LpRecord * r = rec + k;
    logprob_row(logits + (size_t) k * n, n, id, s_row.n_top, &r->lp, r->top_ids, r->top_lp);
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) *(volatile int32_t *)(ring + k) = id;
}

// sentencepiece-style greedy bigram merging, as tensor_processor.cpp:1596-1714 specifies it:
// start from UTF-8 characters, repeatedly merge the adjacent pair whose concatenation is the vocabulary
// entry with the highest score (ties: leftmost), then map pieces to ids, unknown pieces to byte ids (+3).
static void tokenize_pieces(const b200_extra & e, const std::string & text, std::vector<int32_t> & out) {
    struct Piece { int prev, next; size_t off, len; };
    struct Cand { float score; int left, right; size_t len; };
    struct Worse { bool operator()(const Cand & a, const Cand & b) const { return a.score < b.score || (a.score == b.score && a.left > b.left); } };
    std::vector<Piece> ps;
    for (size_t off = 0; off < text.size();) {
        static const size_t lens[16] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};
        size_t n = std::min(text.size() - off, lens[(uint8_t) text[off] >> 4]);
        const int idx = (int) ps.size();
        ps.push_back({idx - 1, off + n == text.size() ? -1 : idx + 1, off, n});
        off += n;
    }
    std::priority_queue<Cand, std::vector<Cand>, Worse> heap;
    auto offer = [&](int l, int r) {
        if (l < 0 || r < 0) return;
        const std::string joined = text.substr(ps[l].off, ps[l].len + ps[r].len);
        auto it = e.token_to_id.find(joined);
        if (it == e.token_to_id.end() || (size_t) it->second >= e.vocab.size()) return;
        heap.push({e.vocab[it->second].second, l, r, joined.size()});
    };
    for (int i = 1; i < (int) ps.size(); i++) offer(i - 1, i);
    while (!heap.empty()) {
        const Cand c = heap.top(); heap.pop();
        Piece & L = ps[c.left]; Piece & R = ps[c.right];
        if (L.len == 0 || R.len == 0 || L.len + R.len != c.len) continue;      // stale candidate
        L.len += R.len; R.len = 0;
        L.next = R.next;
        if (R.next >= 0) ps[R.next].prev = c.left;
        offer(L.prev, c.left);
        offer(c.left, L.next);
    }
    for (int i = ps.empty() ? -1 : 0; i != -1; i = ps[i].next) {
        auto it = e.token_to_id.find(text.substr(ps[i].off, ps[i].len));
        if (it != e.token_to_id.end()) out.push_back(it->second);
        else for (size_t j = 0; j < ps[i].len; j++) out.push_back((int32_t)(uint8_t) text[ps[i].off + j] + 3);
    }
}

}  // namespace b200

extern "C" {

int b200_extra_load(const char * path, int device, b200_extra_t ** out) {
    if (!path || !out) return fail(B200_EINVAL, "b200_extra_load: null argument");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(B200_ENODEV, "no CUDA device visible: no CPU fallback");
    if (device < 0 || device >= ndev) return fail(B200_ENODEV, "device %d out of range", device);
    cudaDeviceProp prop;
    B200_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(B200_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    B200_CUDA(cudaSetDevice(device));
    std::unique_ptr<GgjtFile> fp;
    try { fp.reset(new GgjtFile(path, true)); }
    catch (const std::exception & ex) { return fail(B200_EFILE, "error loading extra layers: %s", ex.what()); }
    GgjtFile & f = *fp;
    // frees the stream and every device allocation if the load fails half-way (a node keeps running after a bad extra-layers file)
    struct ExtraGuard {
        b200_extra * p;
        ~ExtraGuard() {
            if (!p) return;
            b200_slice * c = &p->ctx;
            if (c->stream) cudaStreamSynchronize(c->stream);
            for (void * q : c->allocs) cudaFree(q);
            if (c->ev0) cudaEventDestroy(c->ev0);
            if (c->ev1) cudaEventDestroy(c->ev1);
            if (c->stream) cudaStreamDestroy(c->stream);
            delete p;
        }
    };
    ExtraGuard e_guard{new b200_extra()};
    b200_extra * e = e_guard.p;
    b200_slice * s = &e->ctx;
    s->device = device; s->n_sm = prop.multiProcessorCount;
    s->use_pdl = false; s->use_graph = false;
    B200_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    e->n_vocab = (int) f.n_vocab; e->E = (int) f.n_embd;
    const uint32_t E = f.n_embd, V = f.n_vocab;
    int rc;
    try {
        const GgjtTensor & te = f.get("tok_embeddings.weight", {E, V});
        const GgjtTensor & tn = f.get("norm.weight", {E});
        const GgjtTensor & to = f.get("output.weight", {E, V});
        e->emb_type = (int) te.type; e->out_type = (int) to.type;
        if (!wt_block_quant((int) te.type) && te.type != GT_F16 && te.type != GT_F32 && te.type != GT_Q4_K)
            return fail(B200_EFILE, "tok_embeddings type %u unsupported", te.type);
        if (te.type == GT_Q4_K && E % 256) return fail(B200_EFILE, "Q4_K tok_embeddings needs n_embd %% 256 == 0");
        if (!wt_block_quant((int) to.type) && to.type != GT_F16 && to.type != GT_Q6_K)
            return fail(B200_EFILE, "output.weight type %u unsupported (Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, F16, Q6_K)", to.type);
        if (to.type == GT_Q6_K && E % 256) return fail(B200_EFILE, "Q6_K output.weight needs n_embd %% 256 == 0");
        if (tn.type != GT_F32) return fail(B200_EFILE, "norm.weight must be F32");
        if ((rc = dev_alloc(s, &e->emb_raw, te.nbytes)) || (rc = dev_alloc(s, &e->norm_w, (size_t) E))) return rc;
        B200_CUDA(cudaMemcpyAsync(e->norm_w, f.data(tn), (size_t) E * 4, cudaMemcpyHostToDevice, s->stream));
        std::vector<LoadJob> jobs;
        LoadJob je; je.kind = 2; je.nsrc = 1; je.src[0] = &te; je.raw_dst = e->emb_raw; jobs.push_back(je);
        LoadJob jo; jo.nsrc = 1; jo.src[0] = &to;
        if (to.type == GT_F16) { jo.kind = 1; jo.outf = &e->out_f16; }
        else { jo.kind = 0; jo.mode = 0; jo.G = 1; jo.out = &e->out; }     // Q6_K: the layers' k-quant packing
        jobs.push_back(jo);
        if ((rc = run_load_jobs(s, f, jobs))) return rc;
    } catch (const std::exception & ex) { return fail(B200_EFILE, "error loading extra layers: %s", ex.what()); }
    // fp16 SiLU table is not needed here, but the launch helper wants events
    B200_CUDA(cudaEventCreate(&s->ev0));
    B200_CUDA(cudaEventCreate(&s->ev1));
    e->vocab = std::move(f.vocab);
    for (int i = 0; i < (int) e->vocab.size(); i++) e->token_to_id[e->vocab[i].first] = i;
    *out = e;
    e_guard.p = nullptr;
    return 0;
}

int b200_extra_unload(b200_extra_t * e) {
    if (!e) return fail(B200_EINVAL, "null handle");
    { std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx); }
    b200_slice * s = &e->ctx;
    cudaSetDevice(s->device);
    if (s->stream) cudaStreamSynchronize(s->stream);
    for (void * p : s->allocs) cudaFree(p);
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    for (cudaEvent_t ev : s->prof_ev) cudaEventDestroy(ev);
    if (s->stream) cudaStreamDestroy(s->stream);
    delete e;
    return 0;
}

int b200_extra_dims(b200_extra_t * e, int * n_vocab, int * n_embd) {
    if (!e) return fail(B200_EINVAL, "null handle");
    if (n_vocab) *n_vocab = e->n_vocab;
    if (n_embd) *n_embd = e->E;
    return 0;
}

int b200_extra_embed(b200_extra_t * e, const int32_t * tokens, int n_tokens, float * out) {
    if (!e || !tokens || !out || n_tokens <= 0) return fail(B200_EINVAL, "bad argument");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc = extra_reserve(e, n_tokens);
    if (rc) return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_tok, tokens, (size_t) n_tokens * 4, cudaMemcpyHostToDevice, s->stream));
    k_embed_rows<<<dim3((e->E + 255) / 256, n_tokens), 256, 0, s->stream>>>(e->emb_raw, e->emb_type, e->E, e->d_tok, e->n_vocab, e->d_x);
    B200_CUDA(cudaGetLastError());
    s->launches++;
    B200_CUDA(cudaMemcpyAsync(out, e->d_x, (size_t) n_tokens * e->E * 4, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

// Final RMSNorm + lm_head of n rows of device activations x ([n][n_embd], n <= cap_tokens) into d_logits [n][n_vocab].
// Every output type groups columns, so output.weight streams once for up to 8 rows.  A Q6_K output.weight is packed like
// the layers' Q6_K matrices: k_quant_q8k quantises each row once (RMSNorm fused), then k_gemv_kq<Q6_K> runs the dot.
static int extra_lmhead(b200_extra * e, const float * x, int n) {
    b200_slice * s = &e->ctx;
    if (e->out_type == kWT_F16) {
        GemvF16Args f{}; f.K = e->E; f.x = x; f.ldx = e->E; f.norm_w = e->norm_w; f.N = n;
        f.rows = e->n_vocab; f.W = e->out_f16; f.y = e->d_logits; f.ldy = e->n_vocab;
        return launch_f16<PRO_NORM, EPI_STORE>(s, f);
    }
    GemvArgs g{}; g.W = e->out; g.x = x; g.ldx = e->E; g.norm_w = e->norm_w; g.y = e->d_logits; g.ldy = e->n_vocab;
    g.N = n; g.out_rows = e->n_vocab;
    if (e->out_type == kWT_Q6_K) {
        if (int rc = quant_kq(s, g, true)) return rc;
        return launch_gemv_kq<1, PRO_PREQ, EPI_STORE>(s, g);
    }
    return launch_gemv<1, PRO_NORM, EPI_STORE>(s, g);
}

static int extra_logits_device(b200_extra * e, const float * emb, int n_tokens) {
    b200_slice * s = &e->ctx;
    int rc = extra_reserve(e, n_tokens);
    if (rc) return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_x, emb, (size_t) n_tokens * e->E * 4, cudaMemcpyHostToDevice, s->stream));
    return extra_lmhead(e, e->d_x, n_tokens);
}

int b200_extra_logits(b200_extra_t * e, const float * emb, int n_tokens, int all_logits, float * out) {
    if (!e || !emb || !out || n_tokens <= 0) return fail(B200_EINVAL, "bad argument");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc = extra_logits_device(e, emb, n_tokens);
    if (rc) return rc;
    const size_t V = (size_t) e->n_vocab;
    if (all_logits) B200_CUDA(cudaMemcpyAsync(out, e->d_logits, (size_t) n_tokens * V * 4, cudaMemcpyDeviceToHost, s->stream));
    else B200_CUDA(cudaMemcpyAsync(out, e->d_logits + (size_t)(n_tokens - 1) * V, V * 4, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_extra_next_token(b200_extra_t * e, const float * emb, int n_tokens, int32_t * token) {
    if (!e || !emb || !token || n_tokens <= 0) return fail(B200_EINVAL, "bad argument");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    // only the LAST token's logits decide (get_llm_output + sample_next_token, tensor_processor.cpp:1787-1908); rows of
    // the lm_head are independent, so computing that row alone is the same arithmetic.  The argmax runs on the device:
    // 4 bytes come back instead of n_vocab floats.
    int rc = extra_logits_device(e, emb + (size_t)(n_tokens - 1) * e->E, 1);
    if (rc) return rc;
    k_argmax_first<<<1, 1024, 0, s->stream>>>(e->d_logits, e->n_vocab, e->d_best);
    B200_CUDA(cudaGetLastError());
    s->launches++;
    B200_CUDA(cudaMemcpyAsync(token, e->d_best, 4, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

}  // extern "C"

namespace b200 {

// Every device loop's handles: the slices follow each other in layer order on the extra layers' GPU, with its n_embd,
// outside any pipeline.
static int chain_check(b200_slice * const * slices, int n_slices, const b200_extra * e) {
    for (int i = 0; i < n_slices; i++) {
        const b200_slice * s = slices[i];
        if (s->E != e->E) return fail(B200_EINVAL, "slice %d has n_embd %d, the extra layers %d", i, s->E, e->E);
        if (s->device != e->ctx.device)
            return fail(B200_EINVAL, "slice %d is on device %d, the extra layers on device %d: the loop runs on one GPU", i, s->device, e->ctx.device);
        if (s->pp_world > 1 || s->nccl_comm) return fail(B200_EINVAL, "slice %d is joined to a pipeline", i);
        if (i > 0 && s->first_layer != slices[i - 1]->first_layer + slices[i - 1]->L)
            return fail(B200_EINVAL, "slice %d starts at layer %d, not where slice %d ends (%d)", i, s->first_layer, i - 1,
                        slices[i - 1]->first_layer + slices[i - 1]->L);
    }
    return 0;
}

static int check_tokens(const int32_t * tokens, int n, int n_vocab, const char * what) {
    for (int i = 0; i < n; i++)
        if (tokens[i] < 0 || tokens[i] >= n_vocab) return fail(B200_EINVAL, "%s %d is %d, outside [0, %d)", what, i, tokens[i], n_vocab);
    return 0;
}

// Everything b200_generate_greedy checks before it enqueues anything (the handles' mutexes are held).
static int generate_check(b200_slice * const * slices, int n_slices, const b200_extra * e, const int * sessions,
                          const int * counts, int n_seq, const int32_t * tokens, int n_steps) {
    if (int rc = chain_check(slices, n_slices, e)) return rc;
    if (n_steps < 1) return fail(B200_EINVAL, "n_steps must be positive (got %d)", n_steps);
    int total = 0;
    for (const b200_slice * const * sp = slices; sp < slices + n_slices; sp++)
        if (int rc = check_pass(*sp, sessions, counts, n_seq, &total)) return rc;
    if (int rc = check_tokens(tokens, total, e->n_vocab, "prompt token")) return rc;
    for (int i = 0; i < n_slices; i++)
        for (int k = 0; k < n_seq; k++) {
            const b200_slice * s = slices[i];
            if ((long long) s->past[sessions[k]] + counts[k] + n_steps - 1 > s->n_ctx)
                return fail(B200_ECONTEXT, "context overflow: slice %d session %d n_past %d + %d prompt tokens + %d steps > n_ctx %d",
                            i, sessions[k], s->past[sessions[k]], counts[k], n_steps - 1, s->n_ctx);
        }
    return 0;
}

// The loop borrows the extra layers' stream for every slice (each slice's own stream is idle when it starts), so the whole
// sequence of every token is stream-ordered without events; the slices get their streams back when it ends.
struct StreamLoan {
    std::vector<b200_slice *> slices; std::vector<cudaStream_t> own; cudaStream_t loop;
    StreamLoan(b200_slice * const * s, int n, cudaStream_t st) : slices(s, s + n), loop(st) {
        for (b200_slice * p : slices) { own.push_back(p->stream); p->stream = st; }
    }
    ~StreamLoan() {
        cudaStreamSynchronize(loop);
        for (size_t i = 0; i < slices.size(); i++) slices[i]->stream = own[i];
    }
};

// Everything a sampling call checks about its settings before it enqueues anything.
static int sample_check(const b200_sampling_t * sp, int n_seq, int n_vocab) {
    if (!sp || !sp->seeds) return fail(B200_EINVAL, "null sampling settings or seeds");
    if (!(sp->temperature >= 0) || !std::isfinite(sp->temperature))
        return fail(B200_EINVAL, "temperature must be finite and >= 0 (got %g)", sp->temperature);
    if (!(sp->repeat_penalty > 0) || !std::isfinite(sp->repeat_penalty))
        return fail(B200_EINVAL, "repeat penalty must be finite and > 0 (got %g)", sp->repeat_penalty);
    if (sp->first_draw < 0) return fail(B200_EINVAL, "first_draw must be >= 0 (got %lld)", (long long) sp->first_draw);
    if (sp->top_k < 0) return fail(B200_EINVAL, "top_k must be >= 0 (got %d)", (int) sp->top_k);
    if (!(sp->top_p >= 0)) return fail(B200_EINVAL, "top_p must be >= 0 and not NaN (got %g)", sp->top_p);
    if (!sp->history) return 0;
    if (!sp->history_counts) return fail(B200_EINVAL, "a history needs history_counts");
    for (int k = 0, at = 0; k < n_seq; k++) {
        if (sp->history_counts[k] < 0) return fail(B200_EINVAL, "history count %d is %d", k, sp->history_counts[k]);
        for (int j = 0; j < sp->history_counts[k]; j++, at++)
            if (sp->history[at] < 0 || sp->history[at] >= n_vocab)
                return fail(B200_EINVAL, "history id %d of session %d is %d, outside [0, %d)", j, k, sp->history[at], n_vocab);
    }
    return 0;
}

// Uploads the keys and each row's penalty bitmap (cleared, then the bits of its history) and resets the bad-row word.
static int sample_start(b200_extra * e, const b200_sampling_t * sp, int n_seq) {
    if (int rc = extra_reserve_sample(e, n_seq)) return rc;
    const int nw = (e->n_vocab + 31) / 32;
    std::vector<uint32_t> pen((size_t) n_seq * nw, 0u);
    if (sp->history)
        for (int k = 0, at = 0; k < n_seq; k++)
            for (int j = 0; j < sp->history_counts[k]; j++, at++)
                pen[(size_t) k * nw + (sp->history[at] >> 5)] |= 1u << (sp->history[at] & 31);
    const int none = INT_MAX;
    cudaStream_t st = e->ctx.stream;
    B200_CUDA(cudaMemcpyAsync(e->d_pen, pen.data(), pen.size() * 4, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(e->d_seeds, sp->seeds, (size_t) n_seq * 8, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(e->d_bad, &none, 4, cudaMemcpyHostToDevice, st));
    return 0;
}

// k_sample_rows on the first `rows` rows of d_logits (or of `logits`) with draw first_draw + step; a bad row k is
// recorded as step * rows + k.
static int sample_launch(b200_extra * e, const b200_sampling_t * sp, int rows, int step, int32_t * ids,
                         const float * logits = nullptr) {
    const double dt = sp->temperature + 1e-5;
    SampleArgs a{logits ? logits : e->d_logits, e->n_vocab, dt, sp->repeat_penalty * dt, e->d_seeds, (long long) sp->first_draw + step,
                 e->d_pen, e->d_tok, ids, e->d_bad, step * rows, sp->top_k, sp->top_p};
    k_sample_rows<<<rows, 1024, 0, e->ctx.stream>>>(a);
    B200_CUDA(cudaGetLastError());
    e->ctx.launches++;
    return 0;
}

// Everything a call that returns log-probabilities checks about its outputs before it enqueues anything.
static int lp_check(const b200_logprobs_t * lp, int n_vocab) {
    if (!lp || !lp->lp) return fail(B200_EINVAL, "null log-probability outputs");
    if (lp->n_top < 0 || lp->n_top > std::min(kMaxTop, n_vocab))
        return fail(B200_EINVAL, "n_top %d outside [0, %d]", (int) lp->n_top, std::min(kMaxTop, n_vocab));
    if (lp->n_top > 0 && (!lp->top_ids || !lp->top_lp)) return fail(B200_EINVAL, "n_top %d needs top_ids and top_lp", (int) lp->n_top);
    return 0;
}

// The log-probability scratch for `rows` rows of n_top alternatives.
static int lp_reserve(b200_extra * e, int rows, int n_top) {
    int rc;
    if ((rc = extra_regrow(e, e->d_lp, e->cap_lp, 1, rows)) || (rc = extra_regrow(e, e->d_topi, e->cap_topi, 1, rows * n_top)) ||
        (rc = extra_regrow(e, e->d_topl, e->cap_topl, 1, rows * n_top)))
        return rc;
    return 0;
}

// k_logprob_rows on the first `rows` rows of d_logits, whose ids are ids[0, rows): scratch rows r0 .. r0 + rows - 1.
static int lp_launch(b200_extra * e, int rows, const int32_t * ids, int n_top, size_t r0) {
    k_logprob_rows<<<rows, 1024, 0, e->ctx.stream>>>(e->d_logits, e->n_vocab, ids, n_top, e->d_lp + r0, e->d_topi + r0 * n_top,
                                                     e->d_topl + r0 * n_top);
    B200_CUDA(cudaGetLastError());
    e->ctx.launches++;
    return 0;
}

// Scratch rows [0, rows) to the caller's arrays, in stream order (the caller synchronises).
static int lp_copy_back(b200_extra * e, const b200_logprobs_t * lp, int rows) {
    cudaStream_t st = e->ctx.stream;
    const size_t n = (size_t) rows * lp->n_top;
    B200_CUDA(cudaMemcpyAsync(lp->lp, e->d_lp, (size_t) rows * 8, cudaMemcpyDeviceToHost, st));
    if (n) {
        B200_CUDA(cudaMemcpyAsync(lp->top_ids, e->d_topi, n * 4, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaMemcpyAsync(lp->top_lp, e->d_topl, n * 8, cudaMemcpyDeviceToHost, st));
    }
    return 0;
}

// After the call's synchronise: B200_EINVAL naming the first row that had no distribution.
static int sample_finish(b200_extra * e, int rows, const int * sessions) {
    int bad = INT_MAX;
    B200_CUDA(cudaMemcpy(&bad, e->d_bad, 4, cudaMemcpyDeviceToHost));
    if (bad == INT_MAX) return 0;
    const int step = bad / rows, k = bad % rows;
    if (sessions)
        return fail(B200_EINVAL, "step %d session %d: the logits hold a NaN or +inf, are all -inf or overflow float64 once "
                    "scaled, so they have no distribution (its id is -1; positions have moved)", step, sessions[k]);
    return fail(B200_EINVAL, "row %d: the logits are all -inf or overflow float64 once scaled, so they have no distribution", k);
}

// A guided call's mixing settings (b200_guidance_t's scale and smooth_factor).
struct CfgMix { float scale, sf; };

// The loop of b200_generate_greedy (sp == NULL: argmax, k_argmax_rows) and b200_generate_sample (k_sample_rows), and of
// b200_generate_lp (lp != NULL: k_logprob_rows after each step's draw).  With cfg (b200_generate_cfg), sessions, counts
// and tokens list 2 * n_seq entries, guidance session k being entry n_seq + k: every pass carries both rows of each pair,
// the guidance row fed the id its session drew, and k_cfg_rows turns each pair's logits into the row the draw reads, in
// d_cfg; log-probabilities still read the session's raw row.
static int generate_locked(b200_slice * const * slices, int n_slices, b200_extra * e, const int * sessions,
                           const int * counts, int n_seq, const int32_t * tokens, int n_steps, const b200_sampling_t * sp,
                           int32_t * ids, const b200_logprobs_t * lp, const CfgMix * cfg = nullptr) {
    b200_slice * x = &e->ctx;
    B200_CUDA(cudaSetDevice(x->device));
    const int n_rows = cfg ? 2 * n_seq : n_seq;
    int total = 0;
    for (int k = 0; k < n_rows; k++) total += counts[k];
    int rc;
    if ((rc = extra_reserve(e, total)) || (rc = extra_reserve_ids(e, n_steps * n_seq))) return rc;
    if (lp && (rc = lp_reserve(e, n_steps * n_seq, lp->n_top))) return rc;
    if (cfg && (rc = extra_regrow(e, e->d_cfg, e->cap_cfg, (size_t) e->n_vocab, n_seq))) return rc;
    for (int i = 0; i < n_slices; i++) B200_CUDA(cudaStreamSynchronize(slices[i]->stream));
    if (sp && (rc = sample_start(e, sp, n_seq))) return rc;
    if (cfg && !sp) {                                    // greedy guided rows report a pair without a distribution
        const int none = INT_MAX;
        if ((rc = extra_reserve_sample(e, n_seq))) return rc;
        B200_CUDA(cudaMemcpyAsync(e->d_bad, &none, 4, cudaMemcpyHostToDevice, x->stream));
    }
    B200_CUDA(cudaMemcpyAsync(e->d_tok, tokens, (size_t) total * 4, cudaMemcpyHostToDevice, x->stream));
    {
        StreamLoan loan(slices, n_slices, x->stream);
        for (int step = 0; step < n_steps; step++) {
            // step 0: every session's prompt in one mixed pass; later steps: the id each session produced, one batched
            // step (a single session replays its captured decode graph).  Both are exact mode, as b200_mixed_forward.
            const int N = step == 0 ? total : n_rows;
            k_embed_rows<<<dim3((e->E + 255) / 256, N), 256, 0, x->stream>>>(e->emb_raw, e->emb_type, e->E, e->d_tok, e->n_vocab, e->d_x);
            B200_CUDA(cudaGetLastError());
            x->launches++;
            const float * cur = e->d_x;
            for (int i = 0; i < n_slices; i++) {
                b200_slice * s = slices[i];
                if (step == 0)        rc = pass_locked(s, sessions, counts, n_rows, cur, s->d_out, false);
                else if (n_rows == 1) rc = forward_locked(s, cur, 1, s->d_out, false, sessions[0]);
                else                  rc = pass_locked(s, sessions, nullptr, n_rows, cur, s->d_out, false);
                if (rc) return rc;
                cur = s->d_out;
            }
            if (step == 0 && total > n_rows) {       // each session's last prompt row, packed for the lm_head
                for (int k = 0, end = 0; k < n_rows; k++) {
                    end += counts[k];
                    B200_CUDA(cudaMemcpyAsync(e->d_x + (size_t) k * e->E, cur + (size_t)(end - 1) * e->E, (size_t) e->E * 4,
                                              cudaMemcpyDeviceToDevice, x->stream));
                }
                cur = e->d_x;
            }
            if ((rc = extra_lmhead(e, cur, n_rows))) return rc;
            int32_t * step_ids = e->d_ids + (size_t) step * n_seq;
            if (cfg) {
                // greedy: k_cfg_rows' pick is the id; sampled: k_sample_rows draws from the guided rows
                CfgArgs c{e->d_logits, e->d_logits + (size_t) n_seq * e->n_vocab, e->n_vocab, cfg->scale, cfg->sf, e->d_cfg,
                          sp ? nullptr : e->d_tok, sp ? nullptr : step_ids, sp ? nullptr : e->d_bad, step * n_seq};
                k_cfg_rows<<<n_seq, kCfgThreads, 0, x->stream>>>(c);
                B200_CUDA(cudaGetLastError());
                x->launches++;
                if (sp && (rc = sample_launch(e, sp, n_seq, step, step_ids, e->d_cfg))) return rc;
                // the guidance rows of the next step take the ids their sessions drew
                B200_CUDA(cudaMemcpyAsync(e->d_tok + n_seq, e->d_tok, (size_t) n_seq * 4, cudaMemcpyDeviceToDevice, x->stream));
            } else if (sp) {
                if ((rc = sample_launch(e, sp, n_seq, step, step_ids))) return rc;
            } else {
                k_argmax_rows<<<n_seq, 1024, 0, x->stream>>>(e->d_logits, e->n_vocab, e->d_tok, step_ids);
                B200_CUDA(cudaGetLastError());
                x->launches++;
            }
            if (lp && (rc = lp_launch(e, n_seq, step_ids, lp->n_top, (size_t) step * n_seq))) return rc;
        }
    }
    B200_CUDA(cudaMemcpyAsync(ids, e->d_ids, (size_t) n_steps * n_seq * 4, cudaMemcpyDeviceToHost, x->stream));
    if (lp && (rc = lp_copy_back(e, lp, n_steps * n_seq))) return rc;
    B200_CUDA(cudaStreamSynchronize(x->stream));
    return sp || cfg ? sample_finish(e, n_seq, sessions) : 0;
}

}  // namespace b200

extern "C" {

}  // extern "C"

namespace b200 {

// Every handle's mutex of a device loop, in address order, so that two loops that share handles cannot deadlock.  A handle
// that belongs to a generation stream other than `self` is refused.
static int lock_handles(b200_slice_t * const * slices, int n_slices, b200_extra_t * e,
                        std::vector<std::unique_lock<std::mutex>> & locks, const b200_stream * self = nullptr) {
    std::vector<std::mutex *> mus{&e->mu};
    for (int i = 0; i < n_slices; i++) {
        if (!slices[i]) return fail(B200_EINVAL, "slice %d is a null handle", i);
        mus.push_back(&slices[i]->mu);
    }
    std::sort(mus.begin(), mus.end());
    if (std::adjacent_find(mus.begin(), mus.end()) != mus.end()) return fail(B200_EINVAL, "a slice handle is listed twice");
    for (std::mutex * m : mus) locks.emplace_back(*m);
    if (e->ctx.owner != self) return refuse_owned(&e->ctx);
    for (int i = 0; i < n_slices; i++)
        if (slices[i]->owner != self) return refuse_owned(slices[i]);
    return 0;
}

// Every generation entry: the checks, every handle's mutex, then the loop (greedy when not sampled; log-probabilities when
// want_lp).
static int generate(const char * what, bool sampled, b200_slice_t * const * slices, int n_slices, b200_extra_t * e,
                    const int * sessions, const int * prompt_counts, int n_seq, const int32_t * prompt_tokens, int n_steps,
                    const b200_sampling_t * sp, int32_t * ids, bool want_lp, const b200_logprobs_t * lp) {
    if (!slices || n_slices < 1 || !e || !sessions || !prompt_counts || n_seq < 1 || !prompt_tokens || !ids)
        return fail(B200_EINVAL, "%s: null argument or empty list", what);
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = lock_handles(slices, n_slices, e, locks)) return rc;
    if (int rc = generate_check(slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens, n_steps)) return rc;
    if (sampled)
        if (int rc = sample_check(sp, n_seq, e->n_vocab)) return rc;
    if (want_lp)
        if (int rc = lp_check(lp, e->n_vocab)) return rc;
    return generate_locked(slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens, n_steps, sp, ids,
                           want_lp ? lp : nullptr);
}

// The mixing settings every guided call refuses before it touches a handle.
static int cfg_mix_check(float scale, float sf) {
    if (!std::isfinite(scale) || !(scale > 1.f))
        return fail(B200_EINVAL, "guidance scale must be finite and > 1 (got %g): at 1 guidance is off, so do not ask for it",
                    (double) scale);
    if (!std::isfinite(sf)) return fail(B200_EINVAL, "guidance smooth_factor must be finite (got %g)", (double) sf);
    return 0;
}

// b200_generate_cfg: the guidance checks, then generate_locked over the merged lists (real sessions, then guidance ones),
// whose generate_check covers counts, ids and both contexts' room.
static int generate_cfg(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                        const int * prompt_counts, int n_seq, const int32_t * prompt_tokens, int n_steps,
                        const b200_guidance_t * g, const b200_sampling_t * sp, int32_t * ids, const b200_logprobs_t * lp) {
    const char * what = "b200_generate_cfg";
    if (!slices || n_slices < 1 || !e || !sessions || !prompt_counts || n_seq < 1 || !prompt_tokens || !ids)
        return fail(B200_EINVAL, "%s: null argument or empty list", what);
    if (!g || !g->sessions || !g->prompt_counts || !g->prompt_tokens) return fail(B200_EINVAL, "%s: null guidance", what);
    if (int rc = cfg_mix_check(g->scale, g->smooth_factor)) return rc;
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = lock_handles(slices, n_slices, e, locks)) return rc;
    for (int k = 0; k < n_seq; k++) {
        const int gs = g->sessions[k];
        for (int i = 0; i < n_slices; i++)
            if (gs < 0 || gs >= slices[i]->n_sessions)
                return fail(B200_EINVAL, "guidance session %d outside [0, %d) on slice %d", gs, slices[i]->n_sessions, i);
        for (int j = 0; j < n_seq; j++) {
            if (sessions[j] == gs) return fail(B200_EINVAL, "guidance session %d is also a listed session", gs);
            if (j < k && g->sessions[j] == gs) return fail(B200_EINVAL, "guidance session %d listed twice", gs);
        }
        if (g->prompt_counts[k] < 1)
            return fail(B200_EINVAL, "negative prompt %d has %d ids: it needs at least 1", k, g->prompt_counts[k]);
    }
    if (int rc = generate_check(slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens, n_steps)) return rc;
    int n_prompt = 0, n_neg = 0;
    for (int k = 0; k < n_seq; k++) { n_prompt += prompt_counts[k]; n_neg += g->prompt_counts[k]; }
    if (int rc = check_tokens(g->prompt_tokens, n_neg, e->n_vocab, "negative prompt token")) return rc;
    std::vector<int> all_sessions(sessions, sessions + n_seq), all_counts(prompt_counts, prompt_counts + n_seq);
    all_sessions.insert(all_sessions.end(), g->sessions, g->sessions + n_seq);
    all_counts.insert(all_counts.end(), g->prompt_counts, g->prompt_counts + n_seq);
    std::vector<int32_t> all_tokens(prompt_tokens, prompt_tokens + n_prompt);
    all_tokens.insert(all_tokens.end(), g->prompt_tokens, g->prompt_tokens + n_neg);
    if (int rc = generate_check(slices, n_slices, e, all_sessions.data(), all_counts.data(), 2 * n_seq, all_tokens.data(), n_steps))
        return rc;
    if (sp)
        if (int rc = sample_check(sp, n_seq, e->n_vocab)) return rc;
    if (lp)
        if (int rc = lp_check(lp, e->n_vocab)) return rc;
    const CfgMix mix{g->scale, g->smooth_factor};
    return generate_locked(slices, n_slices, e, all_sessions.data(), all_counts.data(), n_seq, all_tokens.data(), n_steps, sp,
                           ids, lp, &mix);
}

// Rows the scoring loop's lm_head and k_nll_rows take at a time: its logits scratch is kScoreRows x n_vocab floats
// (8 MB at 32000 ids) however long the texts are.  Rows of the lm_head are independent, so the blocks change no bit.
static constexpr int kScoreRows = 64;

// b200_score's passes: the sessions, whole and in list order, packed into passes of at most n_ctx fed rows (the smallest
// n_ctx of the slices).  A session's rows are never split across passes: a mixed pass's rows depend on their segment's
// row length, so only one segment per session gives the rows of a single call over the whole text.
// -> the list index of each pass's first session, then n_seq.
static std::vector<int> score_passes(b200_slice * const * slices, int n_slices, const int * fed, int n_seq) {
    int cap = INT_MAX;
    for (int i = 0; i < n_slices; i++) cap = std::min(cap, slices[i]->n_ctx);
    std::vector<int> starts{0};
    for (int k = 0, rows = 0; k < n_seq; k++) {
        if (rows > 0 && rows + fed[k] > cap) { starts.push_back(k); rows = 0; }
        rows += fed[k];
    }
    starts.push_back(n_seq);
    return starts;
}

// Everything b200_score checks before it enqueues anything (the handles' mutexes are held); fills fed and the passes.
static int score_check(b200_slice * const * slices, int n_slices, const b200_extra * e, const int * sessions,
                       const int * counts, int n_seq, const int32_t * tokens, std::vector<int> & fed,
                       std::vector<int> & starts) {
    if (int rc = chain_check(slices, n_slices, e)) return rc;
    long long total = 0;
    for (int k = 0; k < n_seq; k++) {
        if (counts[k] < 2) return fail(B200_EINVAL, "session %d: scoring needs at least 2 tokens (got %d)", sessions[k], counts[k]);
        fed.push_back(counts[k] - 1);
        total += counts[k];
    }
    starts = score_passes(slices, n_slices, fed.data(), n_seq);
    for (int i = 0; i < n_slices; i++)
        for (size_t p = 0; p + 1 < starts.size(); p++) {
            int rows = 0;
            if (int rc = check_pass(slices[i], sessions + starts[p], fed.data() + starts[p], starts[p + 1] - starts[p], &rows))
                return rc;
        }
    std::vector<char> seen(slices[0]->n_sessions, 0);   // every session is in range on every slice by now
    for (int k = 0; k < n_seq; k++) {
        if (seen[sessions[k]]) return fail(B200_EINVAL, "session %d listed twice", sessions[k]);
        seen[sessions[k]] = 1;
    }
    return check_tokens(tokens, (int) total, e->n_vocab, "token");
}

// Each pass: embed its fed rows, run them through every slice (one segment per session, exact mode), then the lm_head and
// k_nll_rows over the last slice's output in blocks of kScoreRows rows.  The ids go up once, the NLLs come back once.
static int score_locked(b200_slice * const * slices, int n_slices, b200_extra * e, const int * sessions, const int * counts,
                        const std::vector<int> & fed, const std::vector<int> & starts, const int32_t * tokens, double * nll) {
    b200_slice * x = &e->ctx;
    B200_CUDA(cudaSetDevice(x->device));
    const int n_seq = starts.back();
    std::vector<int> pass_rows;
    int R = 0;
    for (size_t p = 0; p + 1 < starts.size(); p++) {
        int rows = 0;
        for (int k = starts[p]; k < starts[p + 1]; k++) rows += fed[k];
        pass_rows.push_back(rows);
        R += rows;
    }
    std::vector<int32_t> ids((size_t) 2 * R);            // the fed ids, then the targets, each grouped by session
    for (int k = 0, at = 0, r = 0; k < n_seq; at += counts[k], k++)
        for (int j = 0; j < fed[k]; j++, r++) { ids[r] = tokens[at + j]; ids[R + r] = tokens[at + j + 1]; }
    int rc;
    if ((rc = extra_reserve(e, kScoreRows)) || (rc = extra_reserve_ids(e, 2 * R)) ||
        (rc = extra_regrow(e, e->d_sx, e->cap_sx, (size_t) e->E, *std::max_element(pass_rows.begin(), pass_rows.end()))) ||
        (rc = extra_regrow(e, e->d_nll, e->cap_nll, 1, R)))
        return rc;
    for (int i = 0; i < n_slices; i++) B200_CUDA(cudaStreamSynchronize(slices[i]->stream));
    B200_CUDA(cudaMemcpyAsync(e->d_ids, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, x->stream));
    {
        StreamLoan loan(slices, n_slices, x->stream);
        for (size_t p = 0, row0 = 0; p + 1 < starts.size(); row0 += pass_rows[p], p++) {
            const int a = starts[p], N = pass_rows[p];
            k_embed_rows<<<dim3((e->E + 255) / 256, N), 256, 0, x->stream>>>(e->emb_raw, e->emb_type, e->E, e->d_ids + row0,
                                                                               e->n_vocab, e->d_sx);
            B200_CUDA(cudaGetLastError());
            x->launches++;
            const float * cur = e->d_sx;
            for (int i = 0; i < n_slices; i++) {
                b200_slice * s = slices[i];
                if ((rc = pass_locked(s, sessions + a, fed.data() + a, starts[p + 1] - a, cur, s->d_out, false))) return rc;
                cur = s->d_out;
            }
            for (int b = 0; b < N; b += kScoreRows) {
                const int nb = std::min(kScoreRows, N - b);
                if ((rc = extra_lmhead(e, cur + (size_t) b * e->E, nb))) return rc;
                k_nll_rows<<<nb, 1024, 0, x->stream>>>(e->d_logits, e->n_vocab, e->d_ids + R + row0 + b, e->d_nll + row0 + b);
                B200_CUDA(cudaGetLastError());
                x->launches++;
            }
        }
    }
    B200_CUDA(cudaMemcpyAsync(nll, e->d_nll, (size_t) R * 8, cudaMemcpyDeviceToHost, x->stream));
    B200_CUDA(cudaStreamSynchronize(x->stream));
    return 0;
}

// ---------------------------------------------------------------- windowed perplexity (b200_perplexity_windows)
// Rows the windowed perplexity's lm_head and k_ppl_rows take at a time: a window's scored rows of one pass (255 at
// n_ctx 512) in one block; the logits scratch is 32 MB at 32000 ids.  Rows of the lm_head are independent.
static constexpr int kPplLmRows = 256;

// perplexity.cpp:37, 48, 103 and 130: the windows, their segments and their scored rows; and the waves.
struct PplPlan { int n_ctx, n_batch, first, n_scored, n_chunk, n_pass, W; };

// Everything b200_perplexity_windows checks before it changes anything (the handles' mutexes are held).
static int ppl_check(b200_slice * const * slices, int n_slices, const b200_extra * e, const int * sessions, int n_sessions,
                     const int32_t * tokens, int n_tokens, int n_ctx, int n_batch, PplPlan & p) {
    if (int rc = chain_check(slices, n_slices, e)) return rc;
    if (n_ctx < 2) return fail(B200_EINVAL, "n_ctx must be at least 2 (got %d)", n_ctx);
    if (n_batch < 1) return fail(B200_EINVAL, "n_batch must be positive (got %d)", n_batch);
    if (n_tokens < 0) return fail(B200_EINVAL, "n_tokens must not be negative (got %d)", n_tokens);
    int pass_rows = INT_MAX;
    for (int i = 0; i < n_slices; i++) {
        const b200_slice * s = slices[i];
        if (n_ctx > s->n_ctx) return fail(B200_ECONTEXT, "window n_ctx %d exceeds slice %d's n_ctx %d", n_ctx, i, s->n_ctx);
        for (int k = 0; k < n_sessions; k++)
            if (sessions[k] < 0 || sessions[k] >= s->n_sessions)
                return fail(B200_EINVAL, "session %d outside [0, %d) on slice %d", sessions[k], s->n_sessions, i);
        pass_rows = std::min(pass_rows, s->n_ctx);
    }
    std::vector<char> seen(slices[0]->n_sessions, 0);
    for (int k = 0; k < n_sessions; k++) {
        if (seen[sessions[k]]) return fail(B200_EINVAL, "session %d listed twice", sessions[k]);
        seen[sessions[k]] = 1;
    }
    if (int rc = check_tokens(tokens, n_tokens, e->n_vocab, "token")) return rc;
    p.n_ctx = n_ctx;
    p.n_batch = std::min(n_batch, n_ctx);
    p.first = std::min(512, n_ctx / 2);
    p.n_scored = n_ctx - 1 - p.first;
    p.n_chunk = n_tokens / n_ctx;
    p.n_pass = (n_ctx + p.n_batch - 1) / p.n_batch;
    p.W = std::min(n_sessions, pass_rows / p.n_batch);     // >= 1: n_batch <= n_ctx <= pass_rows
    return 0;
}

// Sets the slices' fast_pass for the life of the call.
struct FastPass {
    std::vector<b200_slice *> slices;
    FastPass(b200_slice * const * s, int n, bool on) : slices(s, s + n) { for (b200_slice * p : slices) p->fast_pass = on; }
    ~FastPass() { for (b200_slice * p : slices) p->fast_pass = false; }
};

// n sessions back to n_past 0 on every slice, stream-ordered on the loop's stream.
static int ppl_reset(b200_slice * const * slices, int n_slices, const int * sessions, int n) {
    for (int i = 0; i < n_slices; i++)
        for (int k = 0; k < n; k++) {
            b200_slice * s = slices[i];
            B200_CUDA(cudaMemsetAsync(s->d_npast + sessions[k], 0, 4, s->stream));
            s->past[sessions[k]] = 0;
        }
    return 0;
}

// Uploaded ids: the fed ids in the order the passes take them (wave by wave, pass by pass, window by window, so each
// pass's rows are contiguous), every window's id 0 already BOS, then the targets in the layout of terms.  Each pass:
// embed its rows, run them through every slice as one mixed pass (segment p of each window of the wave at positions
// p * n_batch ..), then for each window the lm_head and k_ppl_rows over its scored rows only.
static int ppl_locked(b200_slice * const * slices, int n_slices, b200_extra * e, const int * sessions, int n_sessions,
                      const int32_t * tokens, const PplPlan & P, bool fast, float * terms) {
    b200_slice * x = &e->ctx;
    B200_CUDA(cudaSetDevice(x->device));
    for (int i = 0; i < n_slices; i++) B200_CUDA(cudaStreamSynchronize(slices[i]->stream));
    const size_t n_fed = (size_t) P.n_chunk * P.n_ctx, n_terms = (size_t) P.n_chunk * P.n_scored;
    StreamLoan loan(slices, n_slices, x->stream);
    if (int rc = ppl_reset(slices, n_slices, sessions, n_sessions)) return rc;
    if (n_terms == 0) return 0;
    std::vector<int32_t> ids(n_fed + n_terms);
    size_t at = 0;
    for (int c0 = 0; c0 < P.n_chunk; c0 += P.W)
        for (int p = 0; p < P.n_pass; p++) {
            const int j0 = p * P.n_batch, cp = std::min(P.n_batch, P.n_ctx - j0);
            for (int c = c0; c < std::min(c0 + P.W, P.n_chunk); c++)
                for (int j = j0; j < j0 + cp; j++) ids[at++] = j == 0 ? 1 : tokens[(size_t) c * P.n_ctx + j];   // BOS = 1
        }
    for (int c = 0; c < P.n_chunk; c++)
        for (int j = P.first; j < P.n_ctx - 1; j++) ids[at++] = tokens[(size_t) c * P.n_ctx + j + 1];
    int rc;
    if ((rc = extra_reserve(e, kPplLmRows)) || (rc = extra_reserve_ids(e, (int) ids.size())) ||
        (rc = extra_regrow(e, e->d_sx, e->cap_sx, (size_t) e->E, P.W * P.n_batch)) ||
        (rc = extra_regrow(e, e->d_terms, e->cap_terms, 1, (int) n_terms)))
        return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_ids, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, x->stream));
    FastPass fp(slices, n_slices, fast);
    const int32_t * d_tgt = e->d_ids + n_fed;
    std::vector<int> counts(P.W);
    size_t row0 = 0;
    for (int c0 = 0; c0 < P.n_chunk; c0 += P.W) {
        const int nw = std::min(P.W, P.n_chunk - c0);
        if (c0 > 0 && (rc = ppl_reset(slices, n_slices, sessions, nw))) return rc;
        for (int p = 0; p < P.n_pass; p++) {
            const int j0 = p * P.n_batch, cp = std::min(P.n_batch, P.n_ctx - j0), N = nw * cp;
            std::fill(counts.begin(), counts.end(), cp);
            k_embed_rows<<<dim3((e->E + 255) / 256, N), 256, 0, x->stream>>>(e->emb_raw, e->emb_type, e->E, e->d_ids + row0,
                                                                               e->n_vocab, e->d_sx);
            B200_CUDA(cudaGetLastError());
            x->launches++;
            row0 += N;
            const float * cur = e->d_sx;
            for (int i = 0; i < n_slices; i++) {
                b200_slice * s = slices[i];
                if ((rc = pass_locked(s, sessions, counts.data(), nw, cur, s->d_out, false))) return rc;
                cur = s->d_out;
            }
            // scored rows of this segment: j in [max(first, j0), min(n_ctx - 1, j0 + cp))
            const int a = std::max(P.first, j0), b = std::min(P.n_ctx - 1, j0 + cp);
            for (int w = 0; w < nw; w++)
                for (int j = a; j < b; j += kPplLmRows) {
                    const int nb = std::min(kPplLmRows, b - j);
                    const size_t t0 = (size_t)(c0 + w) * P.n_scored + (j - P.first);
                    if ((rc = extra_lmhead(e, cur + ((size_t) w * cp + (j - j0)) * e->E, nb))) return rc;
                    k_ppl_rows<<<(nb + kPplRows - 1) / kPplRows, kPplThreads, 0, x->stream>>>(e->d_logits, e->n_vocab, nb,
                                                                                           d_tgt + t0, e->d_terms + t0);
                    B200_CUDA(cudaGetLastError());
                    x->launches++;
                }
        }
    }
    if ((rc = ppl_reset(slices, n_slices, sessions, n_sessions))) return rc;
    B200_CUDA(cudaMemcpyAsync(terms, e->d_terms, n_terms * 4, cudaMemcpyDeviceToHost, x->stream));
    B200_CUDA(cudaStreamSynchronize(x->stream));
    return 0;
}

// ---------------------------------------------------------------- speculative decoding (b200_generate_speculative)
// One iteration, with t the last emitted id, m the ids emitted so far and p the target's position (where t goes):
//   draft  a two-row decode pass [token at p - 1, t], then k - 1 replays of its decode step, each followed by its lm_head
//          and a proposal d_i (k_spec_draft_pick);
//   check  the target's decode rows [t, d_1 .. d_k] at p .. p + k, its lm_head over the k + 1 rows and its choice g_j after
//          each row (k_spec_check_pick);
//   accept k_spec_accept keeps g_0 .. g_n, n the longest run with d_i == g_(i-1), and moves both chains' positions.
// The two-row draft pass rewrites the draft's row p - 1 with the token it already holds there (or fills it when the
// previous iteration kept all k proposals, so the draft never ran d_k): every iteration has the same shape.  Everything an
// iteration reads (tokens, positions, draw indices) is on the device, so the host only enqueues.
constexpr int kSpecMaxDraft = 15;
constexpr int kSpecLookahead = 2;           // iterations enqueued beyond the last one the host has seen finish

struct SpecState {
    int m, p, iters, passes, drafted, accepted;
    int32_t ctok[kSpecMaxDraft + 1];        // the checking pass's tokens: t, d_1 .. d_k
    int32_t g[kSpecMaxDraft + 1];           // the target's id after each checking row
    int32_t dtok[2];                        // the draft's two-row pass: the token at p - 1, t
    int32_t dcur;                           // the draft's last proposal, its next single step's token
};

// The sampling settings of one speculative call (sampled == 0: greedy, the argmax of the raw logits)
struct SpecSample { uint64_t seed; double dt, dp; long long first_draw; int top_k; double top_p; int sampled; };

__global__ void k_spec_init(SpecState * st, const int32_t * id0, int32_t prev, int p, int * const * npast_d, int n_d) {
    if (threadIdx.x) return;
    st->m = 1; st->p = p; st->iters = 0; st->passes = 0; st->drafted = 0; st->accepted = 0;
    const int32_t t = *id0;
    st->ctok[0] = t; st->dtok[0] = prev; st->dtok[1] = t;
    for (int i = 0; i < n_d; i++) *npast_d[i] = p - 1;
}

// The draft's proposal d_i: the argmax, or the Sampler with the draw the target takes for the id d_i guesses
// (first_draw + m + i - 1) and the penalty set history + ids[0, m) + d_1 .. d_(i-1): `work` starts each iteration as a copy
// of the emitted ids' bitmap `base` and collects the proposals.
__global__ void __launch_bounds__(1024) k_spec_draft_pick(const float * logits, int n, SpecState * st, int i, SpecSample sp,
                                                          const uint32_t * base, uint32_t * work, int nw) {
    if (sp.sampled && i == 1) {
        for (int w = threadIdx.x; w < nw; w += blockDim.x) work[w] = base[w];
        __syncthreads();
    }
    const int id = sp.sampled ? sample_row(logits, n, work, sp.dt, sp.dp, sp.seed, sp.first_draw + st->m + i - 1, sp.top_k, sp.top_p)
                              : argmax_row(logits, n);
    if (threadIdx.x) return;
    st->dcur = id; st->ctok[i] = id;
    if (sp.sampled && id >= 0) work[id >> 5] |= 1u << (id & 31);
}

// The target's id g_j after checking row j (one block per row): the argmax, or the Sampler with draw first_draw + m + j and
// the penalty set history + ids[0, m) + d_1 .. d_j, which is the plain loop's set for ids[m + j] whenever g_j is kept.
// Row j's bitmap is its own copy of `base` with d_1 .. d_j added, so the sampler's arithmetic is k_sample_rows'.
__global__ void __launch_bounds__(1024) k_spec_check_pick(const float * logits, int n, SpecState * st, SpecSample sp,
                                                          const uint32_t * base, uint32_t * rows, int nw) {
    const int j = blockIdx.x;
    const float * x = logits + (size_t) j * n;
    int id;
    if (sp.sampled) {
        uint32_t * bits = rows + (size_t) j * nw;
        for (int w = threadIdx.x; w < nw; w += blockDim.x) bits[w] = base[w];
        __syncthreads();
        if (threadIdx.x == 0)
            for (int i = 1; i <= j; i++) { const int d = st->ctok[i]; if (d >= 0) bits[d >> 5] |= 1u << (d & 31); }
        __syncthreads();
        id = sample_row(x, n, bits, sp.dt, sp.dp, sp.seed, sp.first_draw + st->m + j, sp.top_k, sp.top_p);
    } else {
        id = argmax_row(x, n);
    }
    if (threadIdx.x == 0) st->g[j] = id;
}

// The log-probabilities of the ids k_spec_accept is about to emit (one block per checking row, launched between
// k_spec_check_pick and it): row j < c, with c as k_spec_accept counts it, writes output row m + j for id g_j; the other
// rows return at once.  Checking rows are decode rows, bit-identical to single-token steps, so these equal the plain
// loop's values.
__global__ void __launch_bounds__(1024) k_spec_logprobs(const float * logits, int n, const SpecState * st, int k, int n_steps,
                                                        int n_top, double * lp, int32_t * top_ids, double * top_lp) {
    const int j = blockIdx.x, m = st->m;
    if (m >= n_steps) return;
    int a = 0;
    while (a < k && st->ctok[a + 1] == st->g[a]) a++;
    if (j >= min(a + 1, n_steps - m)) return;
    const size_t r = (size_t) m + j;
    logprob_row(logits + (size_t) j * n, n, st->g[j], n_top, lp + r, top_ids + r * n_top, top_lp + r * n_top);
}

// Keeps g_0 .. g_n (n the largest j <= k with d_i == g_(i-1) for every i <= j), cut at the budget of n_steps ids, and moves
// every target slice to p + (ids emitted) and every draft slice one row before it.  The host never enqueues an iteration
// the ones in flight could leave without budget; should one start with the budget spent, it emits nothing and puts the
// positions back where it found them.  Then it publishes (iterations done, ids emitted) to the host through mapped memory.
__global__ void k_spec_accept(SpecState * st, int k, int n_steps, int32_t * ids, uint32_t * base, int * bad,
                              int * const * npast_t, int n_t, int * const * npast_d, int n_d, volatile int * progress) {
    if (threadIdx.x) return;
    const int m = st->m;
    if (m < n_steps) {
        int n = 0;
        while (n < k && st->ctok[n + 1] == st->g[n]) n++;
        const int c = min(n + 1, n_steps - m);
        for (int j = 0; j < c; j++) {
            const int id = st->g[j];
            ids[m + j] = id;
            if (id < 0) { if (bad) atomicMin(bad, m + j); }
            else if (base) base[id >> 5] |= 1u << (id & 31);
        }
        st->passes++; st->drafted += k; st->accepted += n;
        const int32_t t = st->g[c - 1];
        st->dtok[0] = st->ctok[c - 1]; st->dtok[1] = t; st->ctok[0] = t;
        st->m = m + c; st->p += c;
    }
    for (int i = 0; i < n_t; i++) *npast_t[i] = st->p;
    for (int i = 0; i < n_d; i++) *npast_d[i] = st->p - 1;
    st->iters++;
    __threadfence_system();
    progress[0] = st->iters; progress[1] = st->m;
}

// One single-token step of slice s for `session`: the decode graph when it is used, as forward_locked runs it.
static int decode_step(b200_slice * s, int session, const float * in, float * out) {
    s->cur = session; s->cols = nullptr;
    if (s->use_graph && !s->profiling) return run_decode_graph(s, in, out, false);
    return enqueue_layers(s, in, 1, out);
}

// decode rows of one session over a chain: -> the last slice's output
static int chain_steps(b200_slice * const * sl, int n, int session, const float * in, int N, const float ** out) {
    for (int i = 0; i < n; i++) {
        b200_slice * s = sl[i];
        int rc = begin_steps(s, session, N);
        if (!rc) rc = enqueue_layers(s, in, N, s->d_out);
        end_pass(s);
        if (rc) return rc;
        in = s->d_out;
    }
    *out = in;
    return 0;
}

static int embed_launch(b200_extra * e, const int32_t * tok, int N, float * out) {
    k_embed_rows<<<dim3((e->E + 255) / 256, N), 256, 0, e->ctx.stream>>>(e->emb_raw, e->emb_type, e->E, tok, e->n_vocab, out);
    B200_CUDA(cudaGetLastError());
    e->ctx.launches++;
    return 0;
}

// Everything b200_generate_speculative checks before it enqueues anything (every mutex is held).
static int spec_check(b200_slice * const * t, int nt, const b200_extra * e, int session, b200_slice * const * d, int nd,
                      const b200_extra * de, int dsession, const int32_t * prompt, int n_prompt, int n_steps, int k,
                      const b200_sampling_t * sp) {
    if (int rc = chain_check(t, nt, e)) return rc;
    if (int rc = chain_check(d, nd, de)) return rc;
    if (de->ctx.device != e->ctx.device)
        return fail(B200_EINVAL, "the draft is on device %d, the target on device %d: the loop runs on one GPU", de->ctx.device, e->ctx.device);
    if (de->n_vocab != e->n_vocab) return fail(B200_EINVAL, "the draft has %d ids, the target %d", de->n_vocab, e->n_vocab);
    if (n_steps < 1) return fail(B200_EINVAL, "n_steps must be positive (got %d)", n_steps);
    if (k < 1 || k > kSpecMaxDraft) return fail(B200_EINVAL, "n_draft %d outside [1, %d]", k, kSpecMaxDraft);
    int total = 0;
    for (int i = 0; i < nt; i++) if (int rc = check_pass(t[i], &session, &n_prompt, 1, &total)) return rc;
    for (int i = 0; i < nd; i++) if (int rc = check_pass(d[i], &dsession, &n_prompt, 1, &total)) return rc;
    if (int rc = check_tokens(prompt, n_prompt, e->n_vocab, "prompt token")) return rc;
    const int past = t[0]->past[session];
    for (int c = 0; c < 2; c++)
        for (int i = 0; i < (c ? nd : nt); i++) {
            const b200_slice * s = c ? d[i] : t[i];
            const int q = s->past[c ? dsession : session];
            if (q != past)
                return fail(B200_EINVAL, "%s slice %d is at n_past %d, target slice 0 at %d: both chains must start at one position",
                            c ? "draft" : "target", i, q, past);
            if ((long long) q + n_prompt + n_steps - 1 + k > s->n_ctx)
                return fail(B200_ECONTEXT, "context overflow: %s slice %d n_past %d + %d prompt tokens + %d steps + %d draft rows > n_ctx %d",
                            c ? "draft" : "target", i, q, n_prompt, n_steps - 1, k, s->n_ctx);
        }
    if (sp) return sample_check(sp, 1, e->n_vocab);
    return 0;
}

static int spec_locked(b200_slice * const * t, int nt, b200_extra * e, int session, b200_slice * const * d, int nd,
                       b200_extra * de, int dsession, const int32_t * prompt, int n_prompt, int n_steps, int k,
                       const b200_sampling_t * sp, int32_t * ids, b200_spec_stats_t * stats, const b200_logprobs_t * lp) {
    b200_slice * x = &e->ctx;
    B200_CUDA(cudaSetDevice(x->device));
    const int V = e->n_vocab, nw = (V + 31) / 32, p0 = t[0]->past[session] + n_prompt, p_final = p0 + n_steps - 1;
    int rc;
    if ((rc = extra_reserve(e, std::max(n_prompt, k + 1))) || (rc = extra_reserve_ids(e, n_steps)) ||
        (rc = extra_reserve(de, std::max(n_prompt, 2))))
        return rc;
    if (lp && (rc = lp_reserve(e, n_steps, lp->n_top))) return rc;
    for (int i = 0; i < nt; i++) B200_CUDA(cudaStreamSynchronize(t[i]->stream));
    for (int i = 0; i < nd; i++) B200_CUDA(cudaStreamSynchronize(d[i]->stream));
    B200_CUDA(cudaStreamSynchronize(de->ctx.stream));
    if (sp && (rc = sample_start(e, sp, 1))) return rc;
    // device scratch: the state, the slices' position counters, the draft's and the checking rows' penalty bitmaps
    const size_t off_ptr = (sizeof(SpecState) + 15) & ~(size_t) 15, off_bits = off_ptr + ((sizeof(int *) * (nt + nd) + 15) & ~(size_t) 15);
    const size_t bytes = off_bits + (sp ? (size_t)(k + 2) * nw * 4 : 0);
    uint8_t * blob = nullptr; int * h_prog = nullptr; int * d_prog = nullptr;
    B200_CUDA(cudaMalloc(&blob, bytes));
    if (cudaHostAlloc(&h_prog, 2 * sizeof(int), cudaHostAllocMapped) != cudaSuccess || cudaHostGetDevicePointer(&d_prog, h_prog, 0) != cudaSuccess) {
        if (h_prog) cudaFreeHost(h_prog);
        cudaFree(blob);
        return fail(B200_ECUDA, "cudaHostAlloc of the speculative loop's progress words failed");
    }
    struct Release { uint8_t * b; int * h; ~Release() { cudaFree(b); cudaFreeHost(h); } } release{blob, h_prog};
    SpecState * st = (SpecState *) blob;
    int ** npast = (int **)(blob + off_ptr);
    uint32_t * work = sp ? (uint32_t *)(blob + off_bits) : nullptr, * rows = sp ? work + nw : nullptr;
    uint32_t * base = sp ? e->d_pen : nullptr;       // sample_start's row: the history, then every emitted id
    std::vector<int *> h_npast;
    for (int i = 0; i < nt; i++) h_npast.push_back(t[i]->d_npast + session);
    for (int i = 0; i < nd; i++) h_npast.push_back(d[i]->d_npast + dsession);
    h_prog[0] = 0; h_prog[1] = 1;
    SpecSample ss{};
    if (sp) {
        ss.sampled = 1; ss.seed = sp->seeds[0]; ss.dt = sp->temperature + 1e-5; ss.dp = sp->repeat_penalty * ss.dt;
        ss.first_draw = sp->first_draw; ss.top_k = sp->top_k; ss.top_p = sp->top_p;
    }
    B200_CUDA(cudaMemcpyAsync(npast, h_npast.data(), h_npast.size() * sizeof(int *), cudaMemcpyHostToDevice, x->stream));
    B200_CUDA(cudaMemcpyAsync(e->d_tok, prompt, (size_t) n_prompt * 4, cudaMemcpyHostToDevice, x->stream));
    B200_CUDA(cudaMemcpyAsync(de->d_tok, prompt, (size_t) n_prompt * 4, cudaMemcpyHostToDevice, x->stream));
    int issued = 0;
    {
        std::vector<b200_slice *> all(t, t + nt);
        all.insert(all.end(), d, d + nd);
        all.push_back(&de->ctx);
        StreamLoan loan(all.data(), (int) all.size(), x->stream);
        // step 0: the prompt, one mixed pass on each chain, as b200_generate_greedy's step 0
        const float * cur = e->d_x;
        if ((rc = embed_launch(e, e->d_tok, n_prompt, e->d_x))) return rc;
        for (int i = 0; i < nt; i++) {
            if ((rc = pass_locked(t[i], &session, &n_prompt, 1, cur, t[i]->d_out, false))) return rc;
            cur = t[i]->d_out;
        }
        if ((rc = extra_lmhead(e, cur + (size_t)(n_prompt - 1) * e->E, 1))) return rc;
        if (sp) { if ((rc = sample_launch(e, sp, 1, 0, e->d_ids))) return rc; }
        else {
            k_argmax_rows<<<1, 1024, 0, x->stream>>>(e->d_logits, V, e->d_tok, e->d_ids);
            B200_CUDA(cudaGetLastError());
            x->launches++;
        }
        if (lp && (rc = lp_launch(e, 1, e->d_ids, lp->n_top, 0))) return rc;
        cur = de->d_x;
        if ((rc = embed_launch(de, de->d_tok, n_prompt, de->d_x))) return rc;
        for (int i = 0; i < nd; i++) {
            if ((rc = pass_locked(d[i], &dsession, &n_prompt, 1, cur, d[i]->d_out, false))) return rc;
            cur = d[i]->d_out;
        }
        k_spec_init<<<1, 32, 0, x->stream>>>(st, e->d_ids, prompt[n_prompt - 1], p0, npast + nt, nd);
        B200_CUDA(cudaGetLastError());
        x->launches++;
        // the iterations: each emits at least one id, so n_steps - 1 of them always suffice.  One more is enqueued only while
        // fewer than kSpecLookahead are in flight and those cannot finish the budget (each emits at most k + 1 ids), so no
        // iteration runs after the last id.
        for (long spins = 0; issued < n_steps - 1;) {
            const int done = ((volatile int *) h_prog)[0], m = ((volatile int *) h_prog)[1];
            if (m >= n_steps) break;
            const int flying = issued - done;
            if (flying >= kSpecLookahead || (long long) m + (long long) flying * (k + 1) >= n_steps) {
                // now and then make sure the device is still running the iterations (b200_stream_read's guard)
                if (++spins % 4096 == 0) {
                    const cudaError_t q = cudaStreamQuery(x->stream);
                    if (q != cudaSuccess && q != cudaErrorNotReady)
                        return fail(B200_ECUDA, "speculative loop: %s", cudaGetErrorString(q));
                    if (q == cudaSuccess && ((volatile int *) h_prog)[0] < issued)
                        return fail(B200_ECUDA, "speculative loop: the device finished an iteration without publishing it");
                }
                std::this_thread::yield();
                continue;
            }
            spins = 0;
            if ((rc = embed_launch(de, st->dtok, 2, de->d_x)) || (rc = chain_steps(d, nd, dsession, de->d_x, 2, &cur)) ||
                (rc = extra_lmhead(de, cur + de->E, 1)))
                return rc;
            k_spec_draft_pick<<<1, 1024, 0, x->stream>>>(de->d_logits, V, st, 1, ss, base, work, nw);
            B200_CUDA(cudaGetLastError());
            x->launches++;
            for (int i = 2; i <= k; i++) {
                if ((rc = embed_launch(de, &st->dcur, 1, de->d_x))) return rc;
                cur = de->d_x;
                for (int j = 0; j < nd; j++) {
                    if ((rc = decode_step(d[j], dsession, cur, d[j]->d_out))) return rc;
                    cur = d[j]->d_out;
                }
                if ((rc = extra_lmhead(de, cur, 1))) return rc;
                k_spec_draft_pick<<<1, 1024, 0, x->stream>>>(de->d_logits, V, st, i, ss, base, work, nw);
                B200_CUDA(cudaGetLastError());
                x->launches++;
            }
            if ((rc = embed_launch(e, st->ctok, k + 1, e->d_x)) || (rc = chain_steps(t, nt, session, e->d_x, k + 1, &cur)) ||
                (rc = extra_lmhead(e, cur, k + 1)))
                return rc;
            k_spec_check_pick<<<k + 1, 1024, 0, x->stream>>>(e->d_logits, V, st, ss, base, rows, nw);
            B200_CUDA(cudaGetLastError());
            if (lp) {
                k_spec_logprobs<<<k + 1, 1024, 0, x->stream>>>(e->d_logits, V, st, k, n_steps, lp->n_top, e->d_lp, e->d_topi, e->d_topl);
                B200_CUDA(cudaGetLastError());
                x->launches++;
            }
            k_spec_accept<<<1, 32, 0, x->stream>>>(st, k, n_steps, e->d_ids, base, sp ? e->d_bad : nullptr, npast, nt,
                                                   npast + nt, nd, d_prog);
            B200_CUDA(cudaGetLastError());
            x->launches += 2;
            issued++;
        }
    }
    SpecState h{};
    B200_CUDA(cudaMemcpyAsync(ids, e->d_ids, (size_t) n_steps * 4, cudaMemcpyDeviceToHost, x->stream));
    if (lp && (rc = lp_copy_back(e, lp, n_steps))) return rc;
    B200_CUDA(cudaMemcpyAsync(&h, st, sizeof(SpecState), cudaMemcpyDeviceToHost, x->stream));
    for (int * q : h_npast) B200_CUDA(cudaMemcpyAsync(q, &p_final, 4, cudaMemcpyHostToDevice, x->stream));
    B200_CUDA(cudaStreamSynchronize(x->stream));
    for (int i = 0; i < nt; i++) t[i]->past[session] = p_final;
    for (int i = 0; i < nd; i++) d[i]->past[dsession] = p_final;
    if (stats) { stats->passes = h.passes; stats->drafted = h.drafted; stats->accepted = h.accepted; }
    return sp ? sample_finish(e, 1, &session) : 0;
}

// b200_generate_speculative: the checks, every handle's mutex of both chains in address order, then the loop.
static int speculative(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int session, b200_slice_t * const * draft,
                       int n_draft_slices, b200_extra_t * draft_e, int draft_session, const int32_t * prompt, int n_prompt,
                       int n_steps, int n_draft, const b200_sampling_t * sp, int32_t * ids, b200_spec_stats_t * stats,
                       bool want_lp, const b200_logprobs_t * lp) {
    if (!slices || n_slices < 1 || !e || !draft || n_draft_slices < 1 || !draft_e || !prompt || n_prompt < 1 || !ids)
        return fail(B200_EINVAL, "b200_generate_speculative: null argument or empty list");
    std::vector<std::mutex *> mus{&e->mu, &draft_e->mu};
    for (int c = 0; c < 2; c++)
        for (int i = 0; i < (c ? n_draft_slices : n_slices); i++) {
            b200_slice * s = c ? draft[i] : slices[i];
            if (!s) return fail(B200_EINVAL, "%s slice %d is a null handle", c ? "draft" : "target", i);
            mus.push_back(&s->mu);
        }
    std::sort(mus.begin(), mus.end());
    if (std::adjacent_find(mus.begin(), mus.end()) != mus.end())
        return fail(B200_EINVAL, "a handle is listed twice (every slice and extra-layers handle of both chains must be distinct)");
    std::vector<std::unique_lock<std::mutex>> locks;
    for (std::mutex * m : mus) locks.emplace_back(*m);
    if (e->ctx.owner) return refuse_owned(&e->ctx);
    if (draft_e->ctx.owner) return refuse_owned(&draft_e->ctx);
    for (int i = 0; i < n_slices; i++) if (slices[i]->owner) return refuse_owned(slices[i]);
    for (int i = 0; i < n_draft_slices; i++) if (draft[i]->owner) return refuse_owned(draft[i]);
    if (int rc = spec_check(slices, n_slices, e, session, draft, n_draft_slices, draft_e, draft_session, prompt, n_prompt,
                            n_steps, n_draft, sp))
        return rc;
    if (want_lp)
        if (int rc = lp_check(lp, e->n_vocab)) return rc;
    return spec_locked(slices, n_slices, e, session, draft, n_draft_slices, draft_e, draft_session, prompt, n_prompt, n_steps,
                       n_draft, sp, ids, stats, want_lp ? lp : nullptr);
}

}  // namespace b200

extern "C" {

int b200_generate_greedy(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                         const int * prompt_counts, int n_seq, const int32_t * prompt_tokens, int n_steps, int32_t * ids) {
    return generate("b200_generate_greedy", false, slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens, n_steps,
                    nullptr, ids, false, nullptr);
}

int b200_generate_sample(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                         const int * prompt_counts, int n_seq, const int32_t * prompt_tokens, int n_steps,
                         const b200_sampling_t * sp, int32_t * ids) {
    return generate("b200_generate_sample", true, slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens, n_steps,
                    sp, ids, false, nullptr);
}

int b200_generate_lp(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                     const int * prompt_counts, int n_seq, const int32_t * prompt_tokens, int n_steps,
                     const b200_sampling_t * sp, int32_t * ids, const b200_logprobs_t * lp) {
    return generate("b200_generate_lp", sp != nullptr, slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens,
                    n_steps, sp, ids, true, lp);
}

int b200_generate_speculative(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int session,
                              b200_slice_t * const * draft, int n_draft_slices, b200_extra_t * draft_e, int draft_session,
                              const int32_t * prompt, int n_prompt, int n_steps, int n_draft, const b200_sampling_t * sp,
                              int32_t * ids, b200_spec_stats_t * stats) {
    return speculative(slices, n_slices, e, session, draft, n_draft_slices, draft_e, draft_session, prompt, n_prompt, n_steps,
                       n_draft, sp, ids, stats, false, nullptr);
}

int b200_generate_speculative_lp(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int session,
                                 b200_slice_t * const * draft, int n_draft_slices, b200_extra_t * draft_e, int draft_session,
                                 const int32_t * prompt, int n_prompt, int n_steps, int n_draft, const b200_sampling_t * sp,
                                 int32_t * ids, b200_spec_stats_t * stats, const b200_logprobs_t * lp) {
    return speculative(slices, n_slices, e, session, draft, n_draft_slices, draft_e, draft_session, prompt, n_prompt, n_steps,
                       n_draft, sp, ids, stats, true, lp);
}

int b200_extra_sample(b200_extra_t * e, const float * logits, int n_rows, const b200_sampling_t * sp, int32_t * ids) {
    if (!e || !logits || n_rows < 1 || !ids) return fail(B200_EINVAL, "b200_extra_sample: null argument or no rows");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    if (int rc = sample_check(sp, n_rows, e->n_vocab)) return rc;
    const size_t V = (size_t) e->n_vocab;
    for (size_t i = 0; i < (size_t) n_rows * V; i++)
        if (std::isnan(logits[i]) || logits[i] == INFINITY)
            return fail(B200_EINVAL, "row %d has a non-finite logit at id %d (%g)", (int)(i / V), (int)(i % V), (double) logits[i]);
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc;
    if ((rc = extra_reserve(e, n_rows)) || (rc = extra_reserve_ids(e, n_rows)) || (rc = sample_start(e, sp, n_rows))) return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_logits, logits, (size_t) n_rows * V * 4, cudaMemcpyHostToDevice, s->stream));
    if ((rc = sample_launch(e, sp, n_rows, 0, e->d_ids))) return rc;
    B200_CUDA(cudaMemcpyAsync(ids, e->d_ids, (size_t) n_rows * 4, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return sample_finish(e, n_rows, nullptr);
}

int b200_score(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions, const int * counts,
               int n_seq, const int32_t * tokens, double * nll) {
    if (!slices || n_slices < 1 || !e || !sessions || !counts || n_seq < 1 || !tokens || !nll)
        return fail(B200_EINVAL, "b200_score: null argument or empty list");
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = lock_handles(slices, n_slices, e, locks)) return rc;
    std::vector<int> fed, starts;
    if (int rc = score_check(slices, n_slices, e, sessions, counts, n_seq, tokens, fed, starts)) return rc;
    return score_locked(slices, n_slices, e, sessions, counts, fed, starts, tokens, nll);
}

int b200_extra_nll(b200_extra_t * e, const float * logits, int n_rows, const int32_t * targets, double * nll) {
    if (!e || !logits || n_rows < 1 || !targets || !nll) return fail(B200_EINVAL, "b200_extra_nll: null argument or no rows");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    if (int rc = check_tokens(targets, n_rows, e->n_vocab, "target")) return rc;
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc;
    if ((rc = extra_reserve(e, n_rows)) || (rc = extra_reserve_ids(e, n_rows)) || (rc = extra_regrow(e, e->d_nll, e->cap_nll, 1, n_rows)))
        return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_logits, logits, (size_t) n_rows * e->n_vocab * 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaMemcpyAsync(e->d_ids, targets, (size_t) n_rows * 4, cudaMemcpyHostToDevice, s->stream));
    k_nll_rows<<<n_rows, 1024, 0, s->stream>>>(e->d_logits, e->n_vocab, e->d_ids, e->d_nll);
    B200_CUDA(cudaGetLastError());
    s->launches++;
    B200_CUDA(cudaMemcpyAsync(nll, e->d_nll, (size_t) n_rows * 8, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_perplexity_windows(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                            int n_sessions, const int32_t * tokens, int n_tokens, int n_ctx, int n_batch, int fast,
                            float * terms) {
    if (!slices || n_slices < 1 || !e || !sessions || n_sessions < 1 || (!tokens && n_tokens > 0) || (!terms && n_tokens > 0))
        return fail(B200_EINVAL, "b200_perplexity_windows: null argument or empty list");
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = lock_handles(slices, n_slices, e, locks)) return rc;
    PplPlan plan;
    if (int rc = ppl_check(slices, n_slices, e, sessions, n_sessions, tokens, n_tokens, n_ctx, n_batch, plan)) return rc;
    return ppl_locked(slices, n_slices, e, sessions, n_sessions, tokens, plan, fast != 0, terms);
}

int b200_extra_ppl_terms(b200_extra_t * e, const float * logits, int n_rows, const int32_t * targets, float * terms) {
    if (!e || !logits || n_rows < 1 || !targets || !terms) return fail(B200_EINVAL, "b200_extra_ppl_terms: null argument or no rows");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    if (int rc = check_tokens(targets, n_rows, e->n_vocab, "target")) return rc;
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc;
    if ((rc = extra_reserve(e, n_rows)) || (rc = extra_reserve_ids(e, n_rows)) || (rc = extra_regrow(e, e->d_terms, e->cap_terms, 1, n_rows)))
        return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_logits, logits, (size_t) n_rows * e->n_vocab * 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaMemcpyAsync(e->d_ids, targets, (size_t) n_rows * 4, cudaMemcpyHostToDevice, s->stream));
    k_ppl_rows<<<(n_rows + kPplRows - 1) / kPplRows, kPplThreads, 0, s->stream>>>(e->d_logits, e->n_vocab, n_rows, e->d_ids, e->d_terms);
    B200_CUDA(cudaGetLastError());
    s->launches++;
    B200_CUDA(cudaMemcpyAsync(terms, e->d_terms, (size_t) n_rows * 4, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_generate_cfg(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                      const int * prompt_counts, int n_seq, const int32_t * prompt_tokens, int n_steps,
                      const b200_guidance_t * g, const b200_sampling_t * sp, int32_t * ids, const b200_logprobs_t * lp) {
    return generate_cfg(slices, n_slices, e, sessions, prompt_counts, n_seq, prompt_tokens, n_steps, g, sp, ids, lp);
}

int b200_extra_cfg(b200_extra_t * e, const float * base, const float * guidance, int n_rows, float scale, float smooth_factor,
                   float * out, int32_t * greedy) {
    if (!e || !base || !guidance || n_rows < 1 || !out) return fail(B200_EINVAL, "b200_extra_cfg: null argument or no rows");
    if (int rc = cfg_mix_check(scale, smooth_factor)) return rc;
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    const size_t V = (size_t) e->n_vocab;
    for (const float * x : {base, guidance})
        for (size_t i = 0; i < (size_t) n_rows * V; i++)
            if (std::isnan(x[i]) || x[i] == INFINITY)
                return fail(B200_EINVAL, "%s row %d has a non-finite logit at id %d (%g)", x == base ? "base" : "guidance",
                            (int)(i / V), (int)(i % V), (double) x[i]);
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc;
    if ((rc = extra_reserve(e, 2 * n_rows)) || (rc = extra_reserve_ids(e, n_rows)) ||
        (rc = extra_regrow(e, e->d_cfg, e->cap_cfg, V, n_rows)))
        return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_logits, base, (size_t) n_rows * V * 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaMemcpyAsync(e->d_logits + (size_t) n_rows * V, guidance, (size_t) n_rows * V * 4, cudaMemcpyHostToDevice, s->stream));
    CfgArgs c{e->d_logits, e->d_logits + (size_t) n_rows * V, e->n_vocab, scale, smooth_factor, e->d_cfg, e->d_ids, nullptr,
              nullptr, 0};
    k_cfg_rows<<<n_rows, kCfgThreads, 0, s->stream>>>(c);
    B200_CUDA(cudaGetLastError());
    s->launches++;
    B200_CUDA(cudaMemcpyAsync(out, e->d_cfg, (size_t) n_rows * V * 4, cudaMemcpyDeviceToHost, s->stream));
    if (greedy) B200_CUDA(cudaMemcpyAsync(greedy, e->d_ids, (size_t) n_rows * 4, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_extra_logprobs(b200_extra_t * e, const float * logits, int n_rows, const int32_t * ids, int n_top, double * lp,
                        int32_t * top_ids, double * top_lp) {
    if (!e || !logits || n_rows < 1 || !ids) return fail(B200_EINVAL, "b200_extra_logprobs: null argument or no rows");
    std::lock_guard<std::mutex> lk(e->mu); B200_UNOWNED(&e->ctx);
    const b200_logprobs_t out{n_top, lp, top_ids, top_lp};
    if (int rc = lp_check(&out, e->n_vocab)) return rc;
    if (int rc = check_tokens(ids, n_rows, e->n_vocab, "id")) return rc;
    b200_slice * s = &e->ctx;
    B200_CUDA(cudaSetDevice(s->device));
    int rc;
    if ((rc = extra_reserve(e, n_rows)) || (rc = extra_reserve_ids(e, n_rows)) || (rc = lp_reserve(e, n_rows, n_top))) return rc;
    B200_CUDA(cudaMemcpyAsync(e->d_logits, logits, (size_t) n_rows * e->n_vocab * 4, cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaMemcpyAsync(e->d_ids, ids, (size_t) n_rows * 4, cudaMemcpyHostToDevice, s->stream));
    if ((rc = lp_launch(e, n_rows, e->d_ids, n_top, 0)) || (rc = lp_copy_back(e, &out, n_rows))) return rc;
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return 0;
}

int b200_extra_tokenize(b200_extra_t * e, const char * prompt, int32_t * out, int cap) {
    if (!e || !prompt) return -B200_EINVAL;
    const std::string text(prompt);
    std::vector<int32_t> ids;
    if (!text.empty()) { ids.push_back(1); tokenize_pieces(*e, text, ids); }      // BOS = 1 (llama_token_bos)
    for (int i = 0; i < (int) ids.size() && i < cap && out; i++) out[i] = ids[i];
    return (int) ids.size();
}

const char * b200_extra_token_text(b200_extra_t * e, int32_t id, int * len) {
    if (!e || id < 0 || id >= (int32_t) e->vocab.size()) { if (len) *len = 0; return nullptr; }
    if (len) *len = (int) e->vocab[id].first.size();
    return e->vocab[id].first.data();
}

}  // extern "C"

// ============================================================================ generation streams (b200_stream_*)
// The generation loop, open-ended: the host schedules one step at a time (who decodes, which queued prompts join), keeps
// up to `lookahead` steps enqueued beyond the oldest one the caller has not read, and learns the ids from a publish ring in
// mapped pinned memory instead of synchronising.  The slices' streams are lent to the extra layers' stream from open to
// close (StreamLoan), so every step is ordered on one stream, as in generate_locked.
#include <deque>

struct b200_stream {
    std::vector<b200_slice *> slices; b200_extra * e = nullptr;
    std::unique_ptr<b200::StreamLoan> loan;
    int max_rows = 0, lookahead = 0, n_sess = 0, rows_cap = 0, nw = 0;   // rows_cap: sessions one step can hold
    int chunk = 0;                        // prefill_chunk: prompt ids per segment (0: the whole prompt)
    // device: per-session sampler slots, penalty bitmaps [n_sess][nw], last ids
    b200::StreamSlot * d_slots = nullptr; uint32_t * d_pen = nullptr; int32_t * d_last = nullptr;
    // mapped pinned, one region per step in flight (lookahead + 1): token specs [max_rows], rows [rows_cap], ids [rows_cap]
    int32_t * h_spec = nullptr; b200::StreamRow * h_rows = nullptr; int32_t * h_ring = nullptr;
    b200::LpRecord * h_lp = nullptr;      // mapped pinned, [regions][rows_cap]: the logprob ring beside h_ring
    struct Sess {
        int state = 0;                    // 0 not in the stream, 1 queued, 2 admitted (its first chunk is enqueued), 3 the
                                          // guidance session of a guided one
        unsigned gen = 0;                 // bumped when the session leaves: rows of steps enqueued before are dropped
        std::vector<int32_t> prompt, stops;
        std::vector<int> old;             // n_past on each slice when it was added
        int fed = 0;                      // prompt ids enqueued; the session decodes once fed == prompt.size()
        int max_tokens = 0, enq = 0, delivered = 0;   // ids enqueued / returned by b200_stream_read
        int n_top = -1;                   // log-probabilities with n_top alternatives; -1: none
        long long first_draw = 0;
        // classifier-free guidance: a guided session names its guidance session (state 3, owner = the guided one), which
        // is fed neg, then the guided session's ids
        int guide = -1, owner = -1;
        std::vector<int32_t> neg;
        int gfed = 0;                     // negative prompt ids enqueued
        float scale = 0.f, sf = 0.f;
    };
    std::vector<Sess> sess;
    std::deque<int> queue;                // sessions whose prompt is not fully enqueued, in add order (the partly fed first)
    // row k: (session, gen); a step without rows carries only non-final chunks and is done when k_stream_mark stores cell 0
    struct Step { int region; std::vector<std::pair<int, unsigned>> rows; size_t next = 0; };
    std::deque<Step> pending;             // enqueued steps whose ids have not all been read (or whose mark has not come)
    long long n_steps = 0, n_rows = 0;    // steps enqueued and the token rows they carried (b200_stream_stats)
    int most_rows = 0;                    // rows of the largest step
};

namespace b200 {

constexpr int kStreamLookahead = 4;

// The session leaves the stream: n_past = old + n_prompt + delivered - 1 (old when nothing was delivered) on every slice,
// host copy now and device copy in stream order, behind any step the device still runs for it.  Those steps' rows are at
// or above the new n_past, so they are unreachable; so are the rows of its prompt chunks when it leaves mid-prefill.
// A guided session's guidance session leaves with it, at old + n_neg + delivered - 1 by the same rule.
static int stream_finish(b200_stream * st, int k) {
    b200_stream::Sess & z = st->sess[k];
    const bool queued = z.fed < (int) z.prompt.size() || (z.guide >= 0 && z.gfed < (int) z.neg.size());
    if (queued) st->queue.erase(std::find(st->queue.begin(), st->queue.end(), k));
    if (z.state == 2) {
        for (int who : {k, z.guide}) {
            if (who < 0) continue;
            const std::vector<int> & old = who == k ? z.old : st->sess[who].old;
            const int n_in = who == k ? (int) z.prompt.size() : (int) z.neg.size();
            for (size_t i = 0; i < st->slices.size(); i++) {
                b200_slice * s = st->slices[i];
                const int p = z.delivered ? old[i] + n_in + z.delivered - 1 : old[i];
                if (s->past[who] == p) continue;
                s->past[who] = p;
                B200_CUDA(cudaMemcpyAsync(s->d_npast + who, &p, 4, cudaMemcpyHostToDevice, st->e->ctx.stream));   // staged at once
            }
        }
    }
    if (z.guide >= 0) { st->sess[z.guide].state = 0; st->sess[z.guide].owner = -1; st->sess[z.guide].gen++; }
    z.state = 0; z.gen++; z.guide = -1;
    return 0;
}

// Schedules and enqueues one step (*did = false when no session has anything to run): every session whose prompt is fully
// fed and that still owes ids decodes one row; then the sessions with prompt ids left, in add order, each get their next
// chunk (the whole prompt when chunk == 0) while the rows fit in max_rows; the first that does not fit ends the step.
// Only a session whose last chunk is in the pass draws, from that chunk's last row.
// A guided session and its guidance session are one unit: a decode row each (both take the guided session's last id),
// and while prefilling, the next non-final chunk of each prompt; a prompt at its final chunk waits until the other's final
// chunk goes in the same step, which draws.  The guided rows come first among the drawing rows, so the lm_head's guidance
// rows and k_cfg_rows' output follow them in order.
static int stream_step(b200_stream * st, bool * did) {
    *did = false;
    struct Entry { int session, count, src; };            // src: the session whose last id a decode row takes; -1: prompt
    struct Draw { int k, gather, gather2; };
    std::vector<Entry> ent;
    std::vector<Draw> guided, plain;
    int N = 0;
    for (int k = 0; k < st->n_sess; k++) {
        const b200_stream::Sess & z = st->sess[k];
        if (z.state == 2 && z.fed == (int) z.prompt.size() && (z.guide < 0 || z.gfed == (int) z.neg.size()) &&
            z.enq < z.max_tokens) {
            ent.push_back({k, 1, k});
            N++;
            if (z.guide < 0) { plain.push_back({k, N - 1, -1}); continue; }
            ent.push_back({z.guide, 1, k});
            N++;
            guided.push_back({k, N - 2, N - 1});
        }
    }
    std::vector<int> fed_now;                             // queued sessions this step feeds
    std::vector<std::pair<int, int>> chunk_now;           // their (prompt, negative prompt) ids this step
    for (int k : st->queue) {
        const b200_stream::Sess & z = st->sess[k];
        const int left = (int) z.prompt.size() - z.fed, c = st->chunk ? std::min(st->chunk, left) : left;
        int cn = 0;
        bool draws = c == left;
        int cp = c;
        if (z.guide >= 0) {
            const int gleft = (int) z.neg.size() - z.gfed;
            cn = st->chunk ? std::min(st->chunk, gleft) : gleft;
            const bool gfinal = cn == gleft;
            draws = draws && gfinal;
            if (!draws) {                                 // a final chunk waits for the other prompt's final chunk
                if (c == left) cp = 0;
                if (gfinal) cn = 0;
            }
        }
        if (N + cp + cn > st->max_rows) break;
        int gather = -1, gather2 = -1;
        if (cp) { ent.push_back({k, cp, -1}); N += cp; gather = N - 1; }
        if (cn) { ent.push_back({z.guide, cn, -1}); N += cn; gather2 = N - 1; }
        fed_now.push_back(k);
        chunk_now.emplace_back(cp, cn);
        if (draws) (z.guide >= 0 ? guided : plain).push_back({k, gather, gather2});
    }
    const int n = (int) ent.size();
    if (n == 0) return 0;
    const int q = (int)(st->n_steps % (st->lookahead + 1));
    int32_t * spec = st->h_spec + (size_t) q * st->max_rows;
    StreamRow * rows = st->h_rows + (size_t) q * st->rows_cap;
    volatile int32_t * ring = st->h_ring + (size_t) q * st->rows_cap;
    b200_stream::Step step{q, {}, 0};
    for (int j = 0, r = 0; j < n; j++) {
        const Entry & en = ent[j];
        if (en.src >= 0) { spec[r++] = ~en.src; continue; }
        // a prompt chunk: the guided session's or its guidance session's, in the order stream_step listed them
        const b200_stream::Sess & owner = st->sess[st->sess[en.session].state == 3 ? st->sess[en.session].owner : en.session];
        const bool neg = st->sess[en.session].state == 3;
        const int at = neg ? owner.gfed : owner.fed;
        const std::vector<int32_t> & src = neg ? owner.neg : owner.prompt;
        for (int i = at; i < at + en.count; i++) spec[r++] = src[i];
    }
    const int n_g = (int) guided.size();
    std::vector<Draw> drawing(guided);
    drawing.insert(drawing.end(), plain.begin(), plain.end());
    bool any_lp = false;
    for (int d = 0; d < (int) drawing.size(); d++) {
        b200_stream::Sess & z = st->sess[drawing[d].k];
        rows[d] = {z.first_draw + z.enq, drawing[d].k, drawing[d].gather, z.n_top, drawing[d].gather2};
        any_lp |= z.n_top >= 0;
        ring[d] = INT32_MIN;
        step.rows.emplace_back(drawing[d].k, z.gen);
    }
    const int n_draw = (int) drawing.size();
    if (n_draw == 0) ring[0] = INT32_MIN;
    b200_extra * e = st->e;
    b200_slice * x = &e->ctx;
    k_stream_tokens<<<(N + 255) / 256, 256, 0, x->stream>>>(spec, st->d_last, N, e->d_tok);
    k_embed_rows<<<dim3((e->E + 255) / 256, N), 256, 0, x->stream>>>(e->emb_raw, e->emb_type, e->E, e->d_tok, e->n_vocab, e->d_x);
    B200_CUDA(cudaGetLastError());
    x->launches += 2;
    // a single session decoding alone replays the slice's captured decode graph; anything else is one pass (all-1 counts:
    // the batched step).  Both are exact mode, as b200_mixed_forward.
    std::vector<int> ses(n), cnt(n);
    for (int j = 0; j < n; j++) { ses[j] = ent[j].session; cnt[j] = ent[j].count; }
    const float * cur = e->d_x;
    int rc;
    for (b200_slice * s : st->slices) {
        if (N == 1 && ent[0].src >= 0) rc = forward_locked(s, cur, 1, s->d_out, false, ses[0]);
        else                           rc = pass_locked(s, ses.data(), cnt.data(), n, cur, s->d_out, false);
        if (rc) return rc;
        cur = s->d_out;
    }
    int32_t * cells = st->h_ring + (size_t) q * st->rows_cap;
    if (n_draw == 0) {
        k_stream_mark<<<1, 1, 0, x->stream>>>(cells);
        B200_CUDA(cudaGetLastError());
        x->launches++;
    } else {
        const int n_lm = n_draw + n_g;                    // the drawing rows, then the guided ones' guidance rows
        if (N > n_lm || n_g) {                            // each drawing session's last row, packed for the lm_head
            k_gather_rows<<<dim3((e->E + 255) / 256, n_draw), 256, 0, x->stream>>>(cur, rows, e->E, e->d_x);
            B200_CUDA(cudaGetLastError());
            x->launches++;
            if (n_g) {
                k_gather_rows<<<dim3((e->E + 255) / 256, n_g), 256, 0, x->stream>>>(cur, rows, e->E, e->d_x + (size_t) n_draw * e->E,
                                                                                    true);
                B200_CUDA(cudaGetLastError());
                x->launches++;
            }
            cur = e->d_x;
        }
        if ((rc = extra_lmhead(e, cur, n_lm))) return rc;
        const size_t V = (size_t) e->n_vocab;
        if (n_g) {
            // one guidance setting per launch: guided rows are grouped by (scale, sf) runs
            for (int d0 = 0; d0 < n_g;) {
                const b200_stream::Sess & z0 = st->sess[drawing[d0].k];
                int d1 = d0 + 1;
                while (d1 < n_g && st->sess[drawing[d1].k].scale == z0.scale && st->sess[drawing[d1].k].sf == z0.sf) d1++;
                CfgArgs c{e->d_logits + d0 * V, e->d_logits + (n_draw + d0) * V, e->n_vocab, z0.scale, z0.sf, e->d_cfg + d0 * V,
                          e->d_ids + d0, nullptr, nullptr, 0};
                k_cfg_rows<<<d1 - d0, kCfgThreads, 0, x->stream>>>(c);
                B200_CUDA(cudaGetLastError());
                x->launches++;
                d0 = d1;
            }
            k_stream_draw<<<n_g, 1024, 0, x->stream>>>(e->d_cfg, e->n_vocab, rows, st->d_slots, st->d_pen, st->d_last, cells,
                                                       e->d_ids);
            B200_CUDA(cudaGetLastError());
            x->launches++;
        }
        if (n_draw > n_g) {
            k_stream_draw<<<n_draw - n_g, 1024, 0, x->stream>>>(e->d_logits + n_g * V, e->n_vocab, rows + n_g, st->d_slots,
                                                                st->d_pen, st->d_last, cells + n_g);
            B200_CUDA(cudaGetLastError());
            x->launches++;
        }
        if (any_lp) {                               // publishes the rows that asked, after their records
            k_stream_logprobs<<<n_draw, 1024, 0, x->stream>>>(e->d_logits, e->n_vocab, rows, st->d_last, cells,
                                                              st->h_lp + (size_t) q * st->rows_cap);
            B200_CUDA(cudaGetLastError());
            x->launches++;
        }
    }
    for (size_t j = 0; j < fed_now.size(); j++) {
        b200_stream::Sess & z = st->sess[fed_now[j]];
        z.state = 2; z.fed += chunk_now[j].first; z.gfed += chunk_now[j].second;
    }
    st->queue.erase(std::remove_if(st->queue.begin(), st->queue.end(), [st](int k) {
        const b200_stream::Sess & z = st->sess[k];
        return z.fed == (int) z.prompt.size() && (z.guide < 0 || z.gfed == (int) z.neg.size());
    }), st->queue.end());
    for (const Draw & d : drawing) st->sess[d.k].enq++;
    st->pending.push_back(std::move(step));
    st->n_steps++; st->n_rows += N; st->most_rows = std::max(st->most_rows, N);
    *did = true;
    return 0;
}

static void stream_free(b200_stream * st) {
    st->loan.reset();                              // waits for the stream, gives the slices their streams back
    for (b200_slice * s : st->slices) s->owner = nullptr;
    if (st->e) st->e->ctx.owner = nullptr;
    cudaFree(st->d_slots); cudaFree(st->d_pen); cudaFree(st->d_last);
    cudaFreeHost(st->h_spec); cudaFreeHost(st->h_rows); cudaFreeHost(st->h_ring); cudaFreeHost(st->h_lp);
    delete st;
}

// Every stream call holds the handles' mutexes, so a call from another thread on one of them is refused at once.
static int stream_lock(b200_stream * st, std::vector<std::unique_lock<std::mutex>> & locks) {
    if (!st) return fail(B200_EINVAL, "null stream");
    if (int rc = lock_handles(st->slices.data(), (int) st->slices.size(), st->e, locks, st)) return rc;
    B200_CUDA(cudaSetDevice(st->e->ctx.device));
    return 0;
}

// b200_stream_read, and with lp != NULL b200_stream_read_lp: record got's log-probabilities from the ring cell beside the
// id's, or NaN and -1 for a session that asked for none.
static int stream_read(b200_stream * st, int32_t * sessions, int32_t * ids, double * lp, int32_t * top_ids, double * top_lp,
                       int cap, int * n_out) {
    *n_out = 0;
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = stream_lock(st, locks)) return rc;
    int got = 0;
    long long spins = 0;
    for (;;) {
        // a chunked stream tops up only while nothing is in hand: its chunk steps fill the device queue, enqueueing a step
        // then waits for the device, and ids already published would wait with it (they would reach the caller in one
        // burst).  A prefill_chunk 0 stream keeps its pacing: a session added between reads joins the same step as before.
        while ((got == 0 || !st->chunk) && (int) st->pending.size() <= st->lookahead) {
            bool did = false;
            if (int rc = stream_step(st, &did)) return rc;
            if (!did) break;
        }
        if (got == cap || st->pending.empty()) break;
        b200_stream::Step & f = st->pending.front();
        const volatile int32_t * ring = st->h_ring + (size_t) f.region * st->rows_cap;
        if (f.rows.empty() && ring[0] != INT32_MIN) { st->pending.pop_front(); spins = 0; continue; }   // a no-draw step ran
        while (f.next < f.rows.size() && got < cap) {
            const int32_t id = ring[f.next];
            if (id == INT32_MIN) break;
            const int k = f.rows[f.next].first;
            const unsigned gen = f.rows[f.next].second;
            f.next++;
            b200_stream::Sess & z = st->sess[k];
            if (z.state != 2 || z.gen != gen) continue;      // a step the device ran past the session's end
            if (lp) {
                std::atomic_thread_fence(std::memory_order_acquire);    // the record was complete before the id was stored
                const LpRecord & r = st->h_lp[(size_t) f.region * st->rows_cap + f.next - 1];
                const int nt = z.n_top;
                lp[got] = nt >= 0 ? r.lp : std::nan("");
                for (int j = 0; j < kMaxTop; j++) {
                    top_ids[(size_t) got * kMaxTop + j] = j < nt ? r.top_ids[j] : -1;
                    top_lp[(size_t) got * kMaxTop + j] = j < nt ? r.top_lp[j] : std::nan("");
                }
            }
            sessions[got] = k; ids[got] = id; got++;
            z.delivered++;
            if (id < 0 || z.delivered == z.max_tokens || std::find(z.stops.begin(), z.stops.end(), id) != z.stops.end())
                if (int rc = stream_finish(st, k)) return rc;
        }
        if (!f.rows.empty() && f.next == f.rows.size()) { st->pending.pop_front(); spins = 0; continue; }
        if (got > 0) break;
        // nothing published yet: poll; now and then make sure the device is still running the steps
        if (++spins % 4096 == 0) {
            const cudaError_t q = cudaStreamQuery(st->e->ctx.stream);
            if (q != cudaSuccess && q != cudaErrorNotReady) return fail(B200_ECUDA, "generation stream: %s", cudaGetErrorString(q));
            if (q == cudaSuccess && ring[f.next] == INT32_MIN)
                return fail(B200_ECUDA, "generation stream: the device finished a step without publishing its id");
        }
        std::this_thread::yield();
    }
    *n_out = got;
    return 0;
}

}  // namespace b200

extern "C" {

int b200_stream_open(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int max_rows, int lookahead,
                     b200_stream_t ** out) {
    return b200_stream_open_ex(slices, n_slices, e, max_rows, lookahead, 0, out);
}

int b200_stream_open_ex(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int max_rows, int lookahead,
                        int prefill_chunk, b200_stream_t ** out) {
    if (!slices || n_slices < 1 || !e || !out) return fail(B200_EINVAL, "b200_stream_open: null argument or no slices");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(B200_ENODEV, "no CUDA device visible: no CPU fallback");
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = lock_handles(slices, n_slices, e, locks)) return rc;
    if (int rc = chain_check(slices, n_slices, e)) return rc;
    int n_ctx = INT_MAX, n_sess = INT_MAX;
    for (int i = 0; i < n_slices; i++) { n_ctx = std::min(n_ctx, slices[i]->n_ctx); n_sess = std::min(n_sess, slices[i]->n_sessions); }
    if (max_rows <= 0) max_rows = n_ctx;
    if (max_rows > n_ctx) return fail(B200_EINVAL, "max_rows %d exceeds the smallest n_ctx %d", max_rows, n_ctx);
    if (prefill_chunk < 0 || prefill_chunk > max_rows)
        return fail(B200_EINVAL, "prefill_chunk %d outside [0, max_rows %d]", prefill_chunk, max_rows);
    if (lookahead <= 0) lookahead = kStreamLookahead;
    if (lookahead > 1024) return fail(B200_EINVAL, "lookahead %d exceeds 1024", lookahead);
    B200_CUDA(cudaSetDevice(e->ctx.device));
    b200_stream * st = new b200_stream();
    st->slices.assign(slices, slices + n_slices); st->e = e;
    st->max_rows = max_rows; st->lookahead = lookahead; st->n_sess = n_sess; st->chunk = prefill_chunk;
    st->rows_cap = std::min(n_sess, max_rows); st->nw = (e->n_vocab + 31) / 32;
    st->sess.resize(n_sess);
    const size_t regions = (size_t) lookahead + 1;
    auto fail_free = [&](int rc) { delete st; return rc; };
    cudaError_t ce = cudaSuccess;
    if ((ce = cudaMalloc(&st->d_slots, sizeof(StreamSlot) * n_sess)) != cudaSuccess ||
        (ce = cudaMalloc(&st->d_pen, (size_t) 4 * st->nw * n_sess)) != cudaSuccess ||
        (ce = cudaMalloc(&st->d_last, (size_t) 4 * n_sess)) != cudaSuccess ||
        (ce = cudaHostAlloc(&st->h_spec, 4 * regions * max_rows, cudaHostAllocMapped)) != cudaSuccess ||
        (ce = cudaHostAlloc(&st->h_rows, sizeof(StreamRow) * regions * st->rows_cap, cudaHostAllocMapped)) != cudaSuccess ||
        (ce = cudaHostAlloc(&st->h_ring, 4 * regions * st->rows_cap, cudaHostAllocMapped)) != cudaSuccess ||
        (ce = cudaHostAlloc(&st->h_lp, sizeof(LpRecord) * regions * st->rows_cap, cudaHostAllocMapped)) != cudaSuccess) {
        cudaFree(st->d_slots); cudaFree(st->d_pen); cudaFree(st->d_last);
        cudaFreeHost(st->h_spec); cudaFreeHost(st->h_rows); cudaFreeHost(st->h_ring); cudaFreeHost(st->h_lp);
        return fail_free(fail(B200_ECUDA, "stream buffers: %s", cudaGetErrorString(ce)));
    }
    if (int rc = extra_reserve(e, max_rows)) { stream_free(st); return rc; }
    for (int i = 0; i < n_slices; i++)
        if (cudaStreamSynchronize(slices[i]->stream) != cudaSuccess) { stream_free(st); return fail(B200_ECUDA, "slice %d: stream failed", i); }
    st->loan.reset(new StreamLoan(slices, n_slices, e->ctx.stream));
    for (int i = 0; i < n_slices; i++) slices[i]->owner = st;
    e->ctx.owner = st;
    *out = st;
    return 0;
}

int b200_stream_add(b200_stream_t * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                    const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop) {
    return b200_stream_add_lp(st, session, prompt, n_prompt, max_tokens, sp, stop_ids, n_stop, -1);
}

}  // extern "C"

namespace b200 {

// The largest step a guided pair's prefill takes under stream_step's rule (chunks of c ids, 0: whole prompts; a final
// chunk waits for the other's).
static int cfg_unit_rows(int n_prompt, int n_neg, int c) {
    if (!c) return n_prompt + n_neg;
    int most = 0;
    for (int a = n_prompt, b = n_neg; a > 0 || b > 0;) {
        const int ca = std::min(c, a), cb = std::min(c, b);
        const bool fa = ca == a, fb = cb == b;
        const int rows = fa && fb ? ca + cb : (fa ? 0 : ca) + (fb ? 0 : cb);
        most = std::max(most, rows);
        if (!(fa && fb)) { if (!fa) a -= ca; if (!fb) b -= cb; } else { a = 0; b = 0; }
    }
    return most;
}

// b200_stream_add_lp, and with guide >= 0 b200_stream_add_cfg.
static int stream_add(b200_stream * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                      const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop, int n_top, int guide,
                      const int32_t * neg, int n_neg, float scale, float sf) {
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = stream_lock(st, locks)) return rc;
    if (session < 0 || session >= st->n_sess) return fail(B200_EINVAL, "session %d outside [0, %d)", session, st->n_sess);
    b200_stream::Sess & z = st->sess[session];
    if (z.state == 3) return fail(B200_EINVAL, "session %d is the guidance session of session %d", session, z.owner);
    if (z.state) return fail(B200_EINVAL, "session %d is already in the stream", session);
    if (guide >= 0 || neg) {
        if (guide < 0 || guide >= st->n_sess) return fail(B200_EINVAL, "guidance session %d outside [0, %d)", guide, st->n_sess);
        if (guide == session) return fail(B200_EINVAL, "session %d cannot be its own guidance session", session);
        if (st->sess[guide].state == 3)
            return fail(B200_EINVAL, "guidance session %d is the guidance session of session %d", guide, st->sess[guide].owner);
        if (st->sess[guide].state) return fail(B200_EINVAL, "guidance session %d is already in the stream", guide);
        if (!neg || n_neg < 1) return fail(B200_EINVAL, "session %d: the negative prompt needs at least one id", session);
        if (int rc = cfg_mix_check(scale, sf)) return rc;
        if (int rc = check_tokens(neg, n_neg, st->e->n_vocab, "negative prompt token")) return rc;
        for (size_t i = 0; i < st->slices.size(); i++) {
            const b200_slice * s = st->slices[i];
            if ((long long) s->past[guide] + n_neg + max_tokens - 1 > s->n_ctx)
                return fail(B200_ECONTEXT, "context overflow: slice %zu guidance session %d n_past %d + %d negative prompt "
                            "tokens + %d steps > n_ctx %d", i, guide, s->past[guide], n_neg, max_tokens - 1, s->n_ctx);
        }
        if (n_prompt >= 1 && cfg_unit_rows(n_prompt, n_neg, st->chunk) > st->max_rows)
            return fail(B200_EINVAL, "session %d: its prompt (%d ids) and negative prompt (%d ids) need a step of %d rows, "
                        "more than max_rows %d", session, n_prompt, n_neg, cfg_unit_rows(n_prompt, n_neg, st->chunk),
                        st->max_rows);
    }
    if (!prompt || n_prompt < 1) return fail(B200_EINVAL, "session %d: the prompt needs at least one id", session);
    if (max_tokens < 1) return fail(B200_EINVAL, "session %d: max_tokens must be positive (got %d)", session, max_tokens);
    if (n_stop < 0 || (n_stop > 0 && !stop_ids)) return fail(B200_EINVAL, "session %d: bad stop list", session);
    const int V = st->e->n_vocab;
    if (int rc = check_tokens(prompt, n_prompt, V, "prompt token")) return rc;
    if (int rc = check_tokens(stop_ids, n_stop, V, "stop id")) return rc;
    if (sp)
        if (int rc = sample_check(sp, 1, V)) return rc;
    if (n_top < -1 || n_top > std::min(kMaxTop, V))
        return fail(B200_EINVAL, "session %d: n_top %d outside [-1, %d]", session, n_top, std::min(kMaxTop, V));
    for (size_t i = 0; i < st->slices.size(); i++) {
        const b200_slice * s = st->slices[i];
        if ((long long) s->past[session] + n_prompt + max_tokens - 1 > s->n_ctx)
            return fail(B200_ECONTEXT, "context overflow: slice %zu session %d n_past %d + %d prompt tokens + %d steps > n_ctx %d",
                        i, session, s->past[session], n_prompt, max_tokens - 1, s->n_ctx);
    }
    if (!st->chunk && n_prompt > st->max_rows)
        return fail(B200_EINVAL, "session %d: a prompt of %d ids exceeds max_rows %d (a prompt is never split)", session, n_prompt, st->max_rows);
    if (guide >= 0) {
        int rc;
        if ((rc = extra_regrow(st->e, st->e->d_cfg, st->e->cap_cfg, (size_t) st->e->n_vocab, st->rows_cap)) ||
            (rc = extra_reserve_ids(st->e, st->rows_cap)))
            return rc;
    }
    // the slot's sampler state, in stream order behind any step still running for an earlier stay of the session
    const double dt = sp ? sp->temperature + 1e-5 : 1.0;
    const StreamSlot slot{sp ? sp->seeds[0] : 0, dt, sp ? sp->repeat_penalty * dt : 1.0, sp ? 1 : 0, sp ? (int) sp->top_k : 0,
                          sp ? sp->top_p : 0.0};
    cudaStream_t cs = st->e->ctx.stream;
    B200_CUDA(cudaMemcpyAsync(st->d_slots + session, &slot, sizeof slot, cudaMemcpyHostToDevice, cs));
    if (sp) {
        std::vector<uint32_t> pen(st->nw, 0u);
        if (sp->history)
            for (int j = 0; j < sp->history_counts[0]; j++) pen[sp->history[j] >> 5] |= 1u << (sp->history[j] & 31);
        B200_CUDA(cudaMemcpyAsync(st->d_pen + (size_t) session * st->nw, pen.data(), pen.size() * 4, cudaMemcpyHostToDevice, cs));
    }
    z.prompt.assign(prompt, prompt + n_prompt);
    z.stops.assign(stop_ids, stop_ids + n_stop);
    z.old.clear();
    for (const b200_slice * s : st->slices) z.old.push_back(s->past[session]);
    z.fed = 0; z.max_tokens = max_tokens; z.enq = 0; z.delivered = 0; z.n_top = n_top;
    z.first_draw = sp ? sp->first_draw : 0;
    z.guide = guide; z.gfed = 0; z.scale = scale; z.sf = sf;
    z.neg.assign(neg, neg + (guide >= 0 ? n_neg : 0));
    if (guide >= 0) {
        b200_stream::Sess & w = st->sess[guide];
        w.state = 3; w.owner = session;
        w.old.clear();
        for (const b200_slice * s : st->slices) w.old.push_back(s->past[guide]);
    }
    z.state = 1;
    st->queue.push_back(session);
    return 0;
}

}  // namespace b200

extern "C" {

int b200_stream_add_lp(b200_stream_t * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                       const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop, int n_top) {
    return stream_add(st, session, prompt, n_prompt, max_tokens, sp, stop_ids, n_stop, n_top, -1, nullptr, 0, 0.f, 0.f);
}

int b200_stream_add_cfg(b200_stream_t * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                        const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop, int n_top, int guidance_session,
                        const int32_t * neg, int n_neg, float scale, float smooth_factor) {
    if (guidance_session < 0) return fail(B200_EINVAL, "guidance session %d outside [0, n_sessions)", guidance_session);
    return stream_add(st, session, prompt, n_prompt, max_tokens, sp, stop_ids, n_stop, n_top, guidance_session, neg, n_neg,
                      scale, smooth_factor);
}

int b200_stream_read(b200_stream_t * st, int32_t * sessions, int32_t * ids, int cap, int * n_out) {
    if (!sessions || !ids || !n_out || cap < 1) return fail(B200_EINVAL, "b200_stream_read: null argument or cap < 1");
    return stream_read(st, sessions, ids, nullptr, nullptr, nullptr, cap, n_out);
}

int b200_stream_read_lp(b200_stream_t * st, int32_t * sessions, int32_t * ids, double * lp, int32_t * top_ids, double * top_lp,
                        int cap, int * n_out) {
    if (!sessions || !ids || !lp || !top_ids || !top_lp || !n_out || cap < 1)
        return fail(B200_EINVAL, "b200_stream_read_lp: null argument or cap < 1");
    return stream_read(st, sessions, ids, lp, top_ids, top_lp, cap, n_out);
}

int b200_stream_cancel(b200_stream_t * st, int session) {
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = stream_lock(st, locks)) return rc;
    if (session < 0 || session >= st->n_sess || st->sess[session].state == 0)
        return fail(B200_EINVAL, "session %d is not in the stream", session);
    if (st->sess[session].state == 3)
        return fail(B200_EINVAL, "session %d is the guidance session of session %d: cancel that one", session,
                    st->sess[session].owner);
    return stream_finish(st, session);
}

int b200_stream_fork(b200_stream_t * st, int src, int dst, int n_keep) {
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = stream_lock(st, locks)) return rc;
    for (int k : {src, dst}) {
        if (k < 0 || k >= st->n_sess) return fail(B200_EINVAL, "session %d outside [0, %d)", k, st->n_sess);
        if (st->sess[k].state == 3)
            return fail(B200_EINVAL, "session %d is the guidance session of session %d", k, st->sess[k].owner);
        if (st->sess[k].state) return fail(B200_EINVAL, "session %d is %s", k, st->sess[k].state == 1 ? "queued" : "active");
    }
    if (src == dst) return fail(B200_EINVAL, "b200_stream_fork: source and destination are both session %d", src);
    for (size_t i = 0; i < st->slices.size(); i++) {
        const int p = st->slices[i]->past[src];
        if (p != st->slices[0]->past[src])
            return fail(B200_EINVAL, "session %d is at position %d on slice 0 and %d on slice %zu", src, st->slices[0]->past[src], p, i);
        if (n_keep < 0 || n_keep > p) return fail(B200_EINVAL, "n_keep %d outside [0, %d] (session %d's position)", n_keep, p, src);
    }
    // in stream order, behind every step still in flight for either session
    for (b200_slice * s : st->slices)
        if (int rc = kv_fork(s, src, &dst, 1, n_keep, st->e->ctx.stream)) return rc;
    return 0;
}

int b200_stream_stats(b200_stream_t * st, int64_t * steps, int64_t * rows, int * most_rows) {
    if (!steps || !rows || !most_rows) return fail(B200_EINVAL, "b200_stream_stats: null argument");
    std::vector<std::unique_lock<std::mutex>> locks;
    if (int rc = stream_lock(st, locks)) return rc;
    *steps = st->n_steps; *rows = st->n_rows; *most_rows = st->most_rows;
    return 0;
}

int b200_stream_close(b200_stream_t * st) {
    int rc;
    {
        std::vector<std::unique_lock<std::mutex>> locks;
        if ((rc = stream_lock(st, locks))) return rc;
        for (int k = 0; k < st->n_sess && !rc; k++)
            if (st->sess[k].state == 1 || st->sess[k].state == 2) rc = stream_finish(st, k);
        if (!rc && cudaStreamSynchronize(st->e->ctx.stream) != cudaSuccess) rc = fail(B200_ECUDA, "generation stream failed");
        st->loan.reset();
        for (b200_slice * s : st->slices) s->owner = nullptr;
        st->e->ctx.owner = nullptr;
    }
    stream_free(st);
    return rc;
}

}  // extern "C"
