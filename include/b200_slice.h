/*
 * b200_slice.h -- C ABI of libb200slice.so, the H100 (sm_90a) slice runtime.
 *
 * Drop-in boundary: these entry points are what the reference's CPython module `llm`
 * (distllm/tensor_processor.cpp:2238-2260) binds for the per-slice forward path, with Python
 * lists replaced by plain float buffers.  Each function cites the reference interface it
 * replaces.  Conventions:
 *   - return 0 on success, a B200_E* code otherwise; no C++ exception crosses the ABI;
 *     b200_last_error() returns a thread-local, human-readable description of the last failure;
 *   - the caller owns every in/out buffer (they are copied, as the reference copies at
 *     tensor_processor.cpp:523 and 798-799); the library owns weights, KV cache and n_past;
 *   - activations are row-major [n_tokens][n_embd] float32 (ggml ne0 = n_embd);
 *   - one handle = one slice on one GPU; calls on a handle are serialised by an internal mutex;
 *   - there is NO CPU fallback: every call fails with B200_ENODEV when no sm_90 device is present.
 */
#ifndef B200_SLICE_H
#define B200_SLICE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_slice b200_slice_t;
typedef struct b200_extra b200_extra_t;

enum {
    B200_OK       = 0,
    B200_EINVAL   = 1,   /* bad argument (null handle, n_tokens <= 0, ...) */
    B200_EFILE    = 2,   /* slice file missing / malformed / unsupported tensor type (layers: Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, F16,
                            or Q4_K / Q6_K matrices in any mix; weight_type is then the first layer's wq type) */
    B200_ENODEV   = 3,   /* no CUDA device, or device is not sm_90 */
    B200_ECUDA    = 4,   /* a CUDA call or kernel failed */
    B200_ECONTEXT = 5,   /* n_past + n_tokens would exceed n_ctx */
    B200_ENCCL    = 6,   /* pipeline hand-off failed */
};

typedef struct b200_slice_info {
    int32_t n_embd, n_head, n_ff, n_layer, first_layer, n_ctx, n_past, weight_type, device;
    int64_t weight_bytes;       /* bytes of slice weights as stored in the reference file */
    int64_t kv_bytes_per_pos;   /* KV-cache bytes appended per position (all layers) */
} b200_slice_info_t;

/* ---- slice lifetime ------------------------------------------------------------------ */

/* llm.load_slice(path)  (tensor_processor.cpp:1995-2009; TransformerSlice ctor 1497-1510).
 * Parses the reference's slice file (GGJT v3 + first_layer, tensor_processor.cpp:152-248),
 * uploads and repacks the weights into HBM, allocates the f16 KV cache for n_ctx positions.
 * n_ctx <= 0 selects the reference default, 512 (vendor examples/common.h:28). */
int b200_slice_load(const char * path, int device, int n_ctx, b200_slice_t ** out);

/* llm.unload_slice()  (tensor_processor.cpp:2023-2030).  Waits for a call that is already inside the library on this
 * handle; the caller must not START another call on the handle concurrently with (or after) unload -- the `llm` module
 * guarantees that with a reference count (csrc/llm_module.cpp). */
int b200_slice_unload(b200_slice_t * s);

/* Create the CUDA context of `device` ahead of the first load (the first CUDA call of a process takes 0.3 s on a 1-GPU
 * box, seconds on an 8-GPU box); optional, lets a caller time b200_slice_load without it. */
int b200_device_init(int device);

/* llm.clear_context()  (tensor_processor.cpp:2012-2021, TransformerSlice::clear_context 1512-1521):
 * n_past = 0; the cache contents become unreachable. */
int b200_slice_clear(b200_slice_t * s);

int b200_slice_info(b200_slice_t * s, b200_slice_info_t * info);

/* Extension (no reference counterpart): move n_past back to `n_past` (<= current) so a benchmark
 * can re-decode positions without re-running the prefill.  Cache rows below n_past stay valid. */
int b200_slice_rewind(b200_slice_t * s, int n_past);

/* ---- the hot path -------------------------------------------------------------------- */

/* llm.propagate_forward(values)  (tensor_processor.cpp:2127-2163 -> TransformerSlice::forward
 * 1523-1544 -> llama_eval_internal 474-809).  `in` and `out` are HOST buffers of
 * n_tokens*n_embd floats; the call copies in (H2D), runs every layer of the slice on the GPU at
 * positions [n_past, n_past+n_tokens), copies out (D2H), and advances n_past. */
int b200_slice_forward(b200_slice_t * s, const float * in, int n_tokens, float * out);

/* Same, with DEVICE buffers on the slice's GPU; asynchronous on the slice's stream unless
 * `sync` != 0.  Used when the activation already lives in HBM (chained slices, benchmarks). */
int b200_slice_forward_device(b200_slice_t * s, const float * d_in, int n_tokens, float * d_out, int sync);

/* ---- sessions and batched steps (additive: SURVEY 8f N3, BASELINE config 5) --------------------
 * The reference holds ONE context per process (tensor_processor.cpp:1491, 1992), so a node serves one sequence at a
 * time.  Here a slice may hold n_sessions independent contexts (own KV cache + own n_past) over the same weights.
 * Session 0 is the context every b200_slice_* call above uses.  Each session behaves exactly like a reference slice
 * of its own: results are bit-identical to a private slice fed the same tokens. */
int b200_slice_load_ex(const char * path, int device, int n_ctx, int n_sessions, b200_slice_t ** out);
/* b200_slice_load_ex with a LoRA adapter merged into the weights on the device, bit-identical to llama.cpp's
 * llama_model_apply_lora_from_file (main --lora / --lora-base, llama.cpp:2846-3124) followed by a plain load.
 * lora_path is a `ggla` v1 file as convert-lora-to-ggml.py writes it.  For each layer matrix W of the slice
 * (attention.wq/wk/wv/wo, feed_forward.w1/w2/w3) with W.loraA (ne [r, K]) and W.loraB (ne [r, rows]):
 *   BA = loraA^T loraB in ggml_vec_dot_f32's AVX2 order, BA *= alpha / r unless that is 1, then
 *   no base:   W = W + BA (quantised W: dequantise, add, requantise with type_traits[W].from_float -- for Q8_0 the AVX2
 *              quantize_row_q8_0, round half to even; F16 W: fp16(fp32(w) + ba));
 *   with base: W = quantise(base + BA), the base tensor (F16: an F16 sum; F32) read in W's place from lora_base_path, a
 *              GGJT v3 slice file of the F16 / F32 model holding the slice's layers (slice_model cuts one).
 * Weight families: Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, F16.  Adapter tensors of layers outside the slice are skipped, so one
 * file serves every slice of a model; an adapter that touches nothing in the slice loads bit-identical to
 * b200_slice_load_ex.  lora_base_path may be NULL.  Everything the adapter contributes is read and checked before the
 * first matrix is repacked; on any error nothing stays loaded.
 * B200_EINVAL: lora_base_path without lora_path.  B200_EFILE, naming the tensor: bad magic or version, a truncated file,
 * r <= 0; a name without the .loraA / .loraB suffix or whose base is not a layer matrix; a lora tensor that is not 2-D or
 * not F32 (llama.cpp asserts on F16); an A / B rank or shape mismatch; rank above 1024; a lone A or B for a matrix of the
 * slice (llama.cpp skips it silently; this refuses it); a targeted Q4_K / Q6_K matrix; a base that lacks the tensor,
 * has another shape, or is not F16 / F32. */
int b200_slice_load_lora(const char * path, int device, int n_ctx, int n_sessions, const char * lora_path,
                         const char * lora_base_path, b200_slice_t ** out);
int b200_session_count(b200_slice_t * s);
int b200_session_n_past(b200_slice_t * s, int session);                      /* -1 on a bad argument */
int b200_session_clear(b200_slice_t * s, int session);                       /* session -1 = every session */
int b200_session_rewind(b200_slice_t * s, int session, int n_past);
/* Session state on the device and off it.  A session's state is its cache rows [0, n_past) and its position; two sessions
 * with the same rows at the same position give bit-identical results (no arithmetic depends on a session's index), so a
 * copied or restored session continues exactly as its source would have.  Each call below takes the handle's mutex, is
 * refused while a generation stream owns the handle, is all-or-nothing (on an error no position moves and no cache byte
 * changes) and synchronises the slice's stream before it returns.
 * b200_session_copy: rows [0, n_keep) of every layer's K and V cache of session src to each of dsts[0, n_dst) in one
 *   launch (each source byte is read once), and each destination's position to n_keep.  Nothing else changes: not src,
 *   not other sessions, not a destination's rows at or above n_keep.  B200_EINVAL: a null handle or dsts, n_dst < 1, a
 *   session outside [0, n_sessions), a destination equal to src or listed twice, n_keep outside [0, n_past of src]. */
int b200_session_copy(b200_slice_t * s, int src, const int * dsts, int n_dst, int n_keep);
/* Bytes b200_session_save writes for the session now: 64 + n_past * kv_bytes_per_pos. */
int b200_session_state_size(b200_slice_t * s, int session, size_t * bytes);
/* The session's state into buf (host memory, pageable or pinned; the copy has finished when the call returns).  Layout,
 * little-endian: a 64-byte header (bytes 0-3 "B2KV", then uint32 version 1, n_embd, n_head, n_layer, first_layer, n_past,
 * zero padding), then the K rows [layer][n_past][n_embd] fp16, then the V rows alike.  *written (may be NULL) = the size.
 * B200_EINVAL: cap < the size (nothing is written), a null handle or buf, a session out of range. */
int b200_session_save(b200_slice_t * s, int session, void * buf, size_t cap, size_t * written);
/* Sets the session's rows [0, n_past) and its position from a blob of b200_session_save, taken from any handle of the same
 * n_embd, n_head, n_layer and first_layer, at any n_ctx >= n_past and any n_sessions.  The blob does not identify the
 * weights: restoring into a different model of the same shape succeeds and is the caller's mistake.  B200_EINVAL (the
 * session untouched): a bad magic, version or shape, n_past > n_ctx, n different from the blob's exact size. */
int b200_session_restore(b200_slice_t * s, int session, const void * buf, size_t n);
int b200_session_forward(b200_slice_t * s, int session, const float * in, int n_tokens, float * out);          /* host buffers */
int b200_session_forward_device(b200_slice_t * s, int session, const float * d_in, int n_tokens, float * d_out, int sync);

/* Decode rows: n_tokens single-token steps of one session in ONE pass, at positions n_past .. n_past + n_tokens - 1.  Row j
 * runs with row length T = n_past + j + 1, as if it were its own step, so the output is bit-identical to n_tokens calls of
 * b200_session_forward with one token each (a prompt chunk's rows are not: their attention follows the chunk's length).
 * The weights stream once for all rows.  The pass table is built on the device from the session's device-side position.
 * Afterwards n_past has advanced by n_tokens.  Fast prefill never applies.  Errors as b200_session_forward. */
int b200_session_forward_steps(b200_slice_t * s, int session, const float * in, int n_tokens, float * out);       /* host buffers */
int b200_session_forward_steps_device(b200_slice_t * s, int session, const float * d_in, int n_tokens, float * d_out, int sync);

/* Throughput mode: ONE token for each of n_seq DISTINCT sessions in a single pass.  in / out are [n_seq][n_embd]; row b
 * belongs to sessions[b] and is processed at that session's own position.  The weights are streamed once for the whole
 * batch; every row's arithmetic is that of its own single-token step, so the result is bit-identical to calling
 * b200_session_forward(sessions[b], row b, 1, ...) for each b.  A session listed twice -> B200_EINVAL. */
int b200_batch_forward(b200_slice_t * s, const int * sessions, int n_seq, const float * in, float * out);      /* host buffers */
int b200_batch_forward_device(b200_slice_t * s, const int * sessions, int n_seq, const float * d_in, float * d_out, int sync);

/* Mixed pass ("chunked prefill"): counts[k] tokens of sessions[k], for n_seq DISTINCT sessions, in a single pass, so a
 * prompt chunk of one session rides along with the decode tokens of the others.  in / out are [sum of counts][n_embd]; rows
 * are grouped by session in list order (the first counts[0] rows belong to sessions[0], the next counts[1] to sessions[1],
 * ...), and session k's rows run at its positions n_past .. n_past + counts[k] - 1.  The weights are streamed once for all
 * rows.  Session k's output rows are bit-identical to b200_session_forward(sessions[k], its rows, counts[k]) on that
 * session alone (so to the reference fed the same chunks); a pass of all-1 counts is b200_batch_forward.  Fast prefill
 * never applies.  All-or-nothing: on an error no position moves and no cache is written.
 *   B200_EINVAL: n_seq < 1, a session out of range or listed twice, a count < 1, sum of counts > n_ctx, a null argument;
 *   B200_ECONTEXT: n_past + counts[k] > n_ctx for some k. */
int b200_mixed_forward(b200_slice_t * s, const int * sessions, const int * counts, int n_seq, const float * in, float * out);   /* host buffers */
int b200_mixed_forward_device(b200_slice_t * s, const int * sessions, const int * counts, int n_seq, const float * d_in, float * d_out,
                              int sync);

/* Fast mode for prefill calls (n_tokens >= min_tokens): the Q4_0 / Q8_0 weight matmuls run on the wgmma tensor cores with
 * the dequantisation fused in (csrc/fastgemm2.cuh; Q4_1, Q5_0, Q5_1, Q4_K / Q6_K and F16 slices ignore the switch and stay exact).
 * NOT bit-exact: operands are rounded to fp16 after the reference's Q8_0 activation quantisation and summed in fp32.
 * Each matmul output is within TAU * sum_k |w16 * x16| of the float64 sum of the same fp16 operands (TAU <= 2^-16, see
 * tests/test_gpu_fast_prefill.py, which also bounds the deviation from exact mode).  The bound is checked per matmul in
 * every kind of call that takes fast mode (tests/test_gpu_fast_prefill_calls.py): prompts from position 0 of up to
 * n_ctx - 1 rows, later chunks of any session (past the 512-row staged attention window too), the last layer of a
 * multi-layer slice, and the mixed passes of b200_perplexity_windows(fast = 1).  Off by default (or
 * B200_FAST_PREFILL=1).  Fast mode never applies to a single-token step, a batched step (b200_batch_forward) or a mixed pass (b200_mixed_forward),
 * whatever min_tokens is: decode always runs in exact mode, on a cache a fast prefill wrote too (the same bits as an
 * exact handle restored from that cache).  A call of fewer than min_tokens rows, or any call after the switch is
 * turned off, is exact mode. */
int b200_slice_set_fast_prefill(b200_slice_t * s, int on, int min_tokens);

/* Block until everything queued on the slice's stream has finished. */
int b200_slice_sync(b200_slice_t * s);

/* Device-side time of the kernels launched by the most recent forward call, in milliseconds
 * (CUDA events on the slice's stream); -1 if none. */
float b200_slice_last_ms(b200_slice_t * s);

/* Record CUDA event `which` (0 = start, 1 = stop) on the slice's stream, and read the time between
 * them: how bench.py times K steps on the stream the kernels are launched on. */
int b200_slice_mark(b200_slice_t * s, int which);
float b200_slice_mark_elapsed_ms(b200_slice_t * s);

/* Per-kernel event timing.  While enabled, forwards run un-graphed with one CUDA-event pair around
 * every launch; _read() returns the summed device time and launch count per kernel class
 * (0 qkv matmul, 1 rope+append, 2 attention, 3 wo matmul, 4 w1/w3 matmul, 5 w2 matmul, 6 advance)
 * since the last read. */
int b200_slice_profile(b200_slice_t * s, int enable);
int b200_slice_profile_read(b200_slice_t * s, float * ms_by_class, int * launches_by_class, int n_class);

/* Number of kernel launches (graph nodes included) issued by this handle so far. */
int64_t b200_slice_launch_count(b200_slice_t * s);

/* Device pointers of the slice's own input / output staging buffers ([n_ctx][n_embd] f32). */
float * b200_slice_dev_in(b200_slice_t * s);
float * b200_slice_dev_out(b200_slice_t * s);

/* Test hook: copy `count` 32-bit words of an internal activation buffer to the host after a forward
 * (0 qkv, 1 att, 2 ffin, 3 gate, 4 xa, 5 xb, 6 q16, 7 k-cache, 8 v-cache, 9 xh: the [n_tokens][K] fp16 activations of
 * the last fast-mode matmul, i.e. w2's input after a fast prefill, 10 the slice's output staging buffer
 * [n_tokens][n_embd] f32, where b200_perplexity_windows' passes leave the last layer's output).  Not part of the
 * drop-in surface. */
int b200_debug_read(b200_slice_t * s, int which, size_t offset_words, size_t count, void * out);

/* Test hook: the packed device bytes of one weight matrix of the slice's layer `layer` (0 = its first).  Block-quantised
 * and k-quant slices: which 0 qkv, 1 wo, 2 w13, 3 w2, 4 / 5 further qkv runs of a k-quant slice; F16 slices: 0..6 = wq,
 * wk, wv, wo, w1, w2, w3.  Every byte of the range is written by the load, so two loads of equal source bytes return
 * equal bytes.  *size (may be null) receives the byte count; count == 0 only queries it. */
int b200_debug_weights(b200_slice_t * s, int layer, int which, size_t offset, size_t count, void * out, size_t * size);

/* Measurement aid (bench.py roofline): while on, a decode step launches only its weight-matmul kernels. */
int b200_debug_skip_attention(b200_slice_t * s, int on);

/* In-kernel %globaltimer timeline of the matmul / attention launches (8 stamps per CTA: [0] entry, [1] dependency
 * resolved, [2] prologue done, [3] exit, [4] last weight copy issued).  _enable(1) re-captures the decode graph with
 * tracing; _read returns the launches recorded so far (class ids as in b200_slice_profile_read). */
int b200_debug_trace_enable(b200_slice_t * s, int on);
int b200_debug_trace_read(b200_slice_t * s, unsigned long long * out, int * cls, int * ctas, int max_launches);

/* ---- layer-slice pipeline over NVLink (one process per GPU) --------------------------- */

/* Join a pipeline of `nranks` slices (rank r holds layer range r of the nodes_map).  `nccl_id`
 * is the 128-byte ncclUniqueId obtained with b200_pipeline_unique_id on rank 0 and distributed
 * by the host (torch.distributed store / TCP).  Replaces the client relaying the activation over
 * TCP between nodes (cli_api/common.py:148-154, control_center.py:224-244) for slices that share
 * one NVSwitch box: the hand-off becomes ONE ncclSend/ncclRecv per hop. */
int b200_pipeline_unique_id(void * id128);
int b200_pipeline_init(b200_slice_t * s, int rank, int nranks, const void * id128);

/* One pipeline step on this rank: rank 0 takes `d_in` (device, may be NULL on other ranks), every
 * rank r>0 receives [n_tokens][n_embd] from r-1, runs its layers, and sends to r+1; the last rank
 * leaves the result in its dev_out buffer and, when `ring` != 0, also sends it to rank 0 (ring = 1: rank 0
 * receives it inside this step into the buffer b200_pipeline_result() returns, closing the token loop; ring = 2: rank 0
 * collects it later, see b200_pipeline_collect). Asynchronous on the slice's stream. */
int b200_pipeline_step(b200_slice_t * s, const float * d_in, int n_tokens, int ring);
/* The same hand-off for one session, and for a batched step (one token for each listed session: [n_seq][n_embd] moves
 * between the slices).  Every rank passes the same session list. */
int b200_pipeline_step_session(b200_slice_t * s, int session, const float * d_in, int n_tokens, int ring);
int b200_pipeline_step_batch(b200_slice_t * s, const int * sessions, int n_seq, const float * d_in, int ring);
/* The same for a mixed pass (b200_mixed_forward): [sum of counts][n_embd] moves between the slices.  Every rank passes the
 * same session and count lists. */
int b200_pipeline_step_mixed(b200_slice_t * s, const int * sessions, const int * counts, int n_seq, const float * d_in, int ring);
/* Peer-memory hand-off (the on-box GPU-native hop): every rank owns a MAILBOX in its HBM (sequence flags + two inbox slots of
 * [n_ctx][n_embd] f32) that its ring neighbours map over NVLink with cudaIpc.  After b200_pipeline_init, each rank
 * exports its 64-byte handle, the host gathers all of them (torch.distributed all_gather, a file, ...) and every rank
 * connects.  From then on b200_pipeline_step* hands the activation over with a store into the next rank's mailbox + a
 * flag, written by the slice's last kernel and polled by the next slice's first kernel inside the captured step graph:
 * no host code, no NCCL kernel between slices.  B200_PP_PEER=0 (or never connecting) keeps ncclSend / ncclRecv. */
int b200_pipeline_mailbox_export(b200_slice_t * s, void * handle64);
int b200_pipeline_mailbox_connect(b200_slice_t * s, const void * handles /* nranks x 64 bytes, rank order */, int nranks);
int b200_pipeline_transport(b200_slice_t * s);   /* 1 = peer mailboxes, 0 = NCCL */
int b200_pipeline_set_transport(b200_slice_t * s, int peer);   /* all ranks alike; 1 only after a successful connect */
/* Measurement aid: bare hand-offs around the ring, no layers; device microseconds per iteration (= nranks hops). */
int b200_pipeline_pingpong(b200_slice_t * s, int n_rows, int iters, float * us_per_iter);
int b200_pipeline_error(b200_slice_t * s);       /* non-zero: a mailbox poll timed out (8 s) on this rank */

/* Throughput mode (BASELINE config 5): a step issued with ring = 2 sends the last slice's output to rank 0 but rank 0 does
 * not wait for it inside the step; it collects the results later, in issue order, with b200_pipeline_collect (rank 0 only;
 * a no-op elsewhere).  Rank 0 can so issue steps for several sessions back to back and every slice stays busy. */
int b200_pipeline_collect(b200_slice_t * s, int n_rows, float * d_dst /* NULL: the pipeline result buffer */);

/* Device pointer of the pipeline's final activation: on rank 0 after a ring step the last slice's output, else dev_out. */
float * b200_pipeline_result(b200_slice_t * s);
int b200_pipeline_destroy(b200_slice_t * s);

/* ---- client-side extra layers (tok_embeddings / norm / output), next-row N1 ------------ */

/* Replace get_inputs / get_llm_output / sample_next_token (tensor_processor.cpp:1717-1908),
 * which re-read the extra-layers file on every call, with a resident copy. */
int b200_extra_load(const char * path, int device, b200_extra_t ** out);
int b200_extra_unload(b200_extra_t * e);
int b200_extra_dims(b200_extra_t * e, int * n_vocab, int * n_embd);
/* llm.prepare_embeddings(path, tokens) -> [n_tokens][n_embd] (host). */
int b200_extra_embed(b200_extra_t * e, const int32_t * tokens, int n_tokens, float * out);
/* llm.get_logits(path, emb, all_logits) -> [n_tokens or 1][n_vocab] (host). */
int b200_extra_logits(b200_extra_t * e, const float * emb, int n_tokens, int all_logits, float * out);
/* llm.get_next_token(path, emb): argmax of the last token's logits (first maximum wins). */
int b200_extra_next_token(b200_extra_t * e, const float * emb, int n_tokens, int32_t * token);
/* Greedy generation on the device: the client's loop (cli_api/common.py:94-111 with get_next_token,
 * tensor_processor.cpp:1894-1908) for n_seq sessions of a model whose slices all live on one GPU.
 * Step 0 feeds each session its prompt (one mixed pass), every later step feeds each session the id it
 * produced (one batched step); after each step the extra layers' norm + lm_head + argmax pick the next id.
 * ids: [n_steps][n_seq].  Session k's ids equal a single-session run, which equals the host loop
 * (b200_extra_embed -> b200_session_forward on each slice -> b200_extra_next_token) with fast prefill off.
 *   - slices: in layer order, each starting where the one before ends; prompt_tokens: sum of prompt_counts ids, grouped
 *     by session in list order.  Each session continues from its current position; afterwards its n_past is
 *     old + prompt_counts[k] + n_steps - 1 on every slice.
 *   - The host enqueues the whole loop and synchronises once.  Every step runs in exact mode (fast prefill never applies).
 *   - Every handle's mutex is held for the call, taken in address order.
 *   - All-or-nothing: on an error no position moves and no cache is written.
 *     B200_EINVAL: a null argument, slices not contiguous in layer order, a slice of another n_embd than the extra layers,
 *     handles on different devices, a handle listed twice or joined to a pipeline, a session out of range or listed
 *     twice, a prompt count < 1, a token id outside [0, n_vocab), n_steps < 1;
 *     B200_ECONTEXT: n_past + prompt_counts[k] + n_steps - 1 > n_ctx on some slice. */
int b200_generate_greedy(b200_slice_t * const * slices, int n_slices, b200_extra_t * e,
                         const int * sessions, const int * prompt_counts, int n_seq,
                         const int32_t * prompt_tokens, int n_steps, int32_t * ids);
/* Sampling settings of the client's Sampler (cli_api/common.py:64-86) for n_seq sessions or rows. */
typedef struct b200_sampling {
    double temperature;          /* >= 0, finite */
    double repeat_penalty;       /* > 0, finite */
    const uint64_t * seeds;      /* [n_seq]: Philox4x64-10 key (seeds[k], 0) = numpy.random.Philox(key=seeds[k]) */
    int64_t first_draw;          /* draws each stream has already given (0 = fresh generator) */
    const int32_t * history;     /* NULL, or ids already sampled, grouped by session: history_counts[k] for session k */
    const int * history_counts;
    int32_t top_k;               /* >= 0; 0 (or >= n_vocab): no top-k cut */
    double top_p;                /* >= 0, not NaN; 0 (or >= 1): no top-p cut */
} b200_sampling_t;
/* Sampled generation on the device: b200_generate_greedy's loop with the client's Sampler in place of the argmax.
 * For each row of logits x, with prev = the session's history plus the ids this call has drawn for it so far:
 *   y_i = x_i / d_i in float64, d_i = repeat_penalty * (T + 1e-5) if i is in prev, else T + 1e-5;
 *   p = softmax(y); the id is the first i with cumsum(p)[i] > u, u = draw (first_draw + step) of session k's
 *   Philox4x64-10 stream as Generator.random() makes it: (word >> 11) * 2^-53.
 * So client.Sampler(T, rp, rng=numpy.random.Generator(numpy.random.Philox(key=seeds[k]))) is the host twin, draw for
 * draw; ids can differ from it only where u lies within ~1e-12 of a CDF boundary (the last ulp of exp and the summation
 * order).  On the device there is no such freedom: a session's ids are the same alone, in a batch, or split across calls
 * (a call with the earlier ids as history, first_draw = their count and the last id as prompt continues another).
 * An id whose probability is exactly 0 is never chosen.
 * Truncation (top_k, top_p; llama.cpp's order and rule), applied per row before the draw:
 *   1. rank the ids by y descending, equal y lower id first (y, not x: the penalty can reorder ids);
 *   2. top-k: K = the first top_k ranked ids (all ids when top_k is 0 or >= n_vocab);
 *   3. top-p: with w_i = exp(y_i - max y) and S_K = sum of w over K, an id of K is kept iff the weight ranked strictly
 *      before it within K is < top_p * S_K; so the top-ranked id is always kept (no cut when top_p is 0 or >= 1);
 *   4. the draw above, unchanged (same u, same id order), on the weights w_i * [i kept].
 * The kept set is a prefix of the ranking, so on the device it is one threshold per row: a key tau (an order-preserving
 * transform of y) and an id cut c; i is kept iff key_i > tau or key_i == tau and i <= c.  The top-p masses are sums of
 * w in fixed point (exact integers, so they do not depend on the order of summation) with an error of at most
 * n_vocab * 2^(floor(log2 n_vocab) - 64) * S_K (2.8e-11 S_K at 32000 ids).  With both off the call runs the untruncated
 * arithmetic; exclusions of ids whose weight is already 0 change no bit.  client.Sampler(T, rp, rng, top_k, top_p) is
 * the host twin; beyond the draw's own ~1e-12, its ids may differ only where its mass before the last kept id or the
 * first dropped one lies within ~1e-10 S_K of top_p * S_K.
 * Everything else, including the error codes, is as b200_generate_greedy; B200_EINVAL also covers a null sp or seeds,
 * temperature < 0 or not finite, repeat_penalty <= 0 or not finite, first_draw < 0, history without history_counts, a
 * history count < 0, a history id outside [0, n_vocab), top_k < 0 and top_p NaN or < 0, and those leave every position
 * unchanged.
 * A row whose logits hold a NaN or +inf, are all -inf, or scale past the float64 range has no distribution (numpy
 * raises "probabilities contain NaN"): its id is -1, the rest of the loop still runs, and the call returns B200_EINVAL
 * naming the first such step and session.  The positions HAVE moved by then, as after a successful call. */
int b200_generate_sample(b200_slice_t * const * slices, int n_slices, b200_extra_t * e,
                         const int * sessions, const int * prompt_counts, int n_seq,
                         const int32_t * prompt_tokens, int n_steps, const b200_sampling_t * sp, int32_t * ids);
/* Speculative decoding on the device, for one session: a draft model proposes n_draft ids, one pass of decode rows of the
 * target (b200_session_forward_steps) checks them, and the longest agreeing prefix is kept.
 *   - Ids: ids[0, n_steps) equal what b200_generate_greedy (sp NULL) or b200_generate_sample (same sp; seeds[0] and
 *     history_counts[0] for this session) writes for this session alone with the same prompt and n_steps, bit for bit,
 *     whatever the draft is.  The draft only decides how many target passes it takes.
 *   - Each iteration: the draft runs n_draft single-token steps from the last emitted id t (greedy: the argmax; sampled:
 *     proposal d_i guesses ids[m + i - 1] and takes that id's draw, first_draw + m + i - 1, with the penalty set history +
 *     ids[0, m) + d_1 .. d_(i-1)); the target runs rows [t, d_1 .. d_k] and chooses g_j after row j with draw
 *     first_draw + m + j and penalty set history + ids[0, m) + d_1 .. d_j; g_0 .. g_n are emitted, n the largest j with
 *     d_i == g_(i-1) for every i <= j.  Step 0 is the prompt: one mixed pass on each chain, as b200_generate_greedy.
 *   - Positions: every slice of both chains must start at one n_past (else B200_EINVAL); afterwards all are at
 *     old + n_prompt + n_steps - 1, as after b200_generate_greedy.  So a second call with prompt = [last id] (sampled: with
 *     the earlier ids as history and first_draw = their count) continues the run exactly.
 *   - Draft chain: its own slices and extra layers on the target's GPU; its n_embd may differ, its n_vocab must equal the
 *     target's.  Every handle of both chains must be distinct.
 *   - The host enqueues iterations without a round trip (positions, tokens and draw indices live on the device), at most 2
 *     beyond the last one it has seen finish (a counter in mapped memory) and none that the iterations in flight could leave
 *     without budget, and synchronises once at the end.  A device error while it waits is B200_ECUDA.
 *   - Locking, chain checks, stream ownership and all-or-nothing errors are as b200_generate_greedy.  Also B200_EINVAL for
 *     n_draft outside [1, 15], a null draft or draft_e, a vocabulary mismatch or unequal starting positions, and
 *     B200_ECONTEXT when n_past + n_prompt + n_steps - 1 + n_draft > n_ctx on any slice of either chain: a check can write
 *     up to n_draft rows past the last kept one (rows nothing reads afterwards).
 *   - stats (may be NULL): passes = target checking passes, drafted = proposals made (passes * n_draft), accepted =
 *     proposals that matched the target's choice (including matches past the budget's end).
 *   - A row with no distribution behaves as in b200_generate_sample: the same ids including -1, and B200_EINVAL naming
 *     the first such step. */
typedef struct b200_spec_stats { int32_t passes, drafted, accepted; } b200_spec_stats_t;
int b200_generate_speculative(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int session,
                              b200_slice_t * const * draft, int n_draft_slices, b200_extra_t * draft_e, int draft_session,
                              const int32_t * prompt, int n_prompt, int n_steps, int n_draft,
                              const b200_sampling_t * sp /* NULL: greedy */, int32_t * ids, b200_spec_stats_t * stats);
/* The sampling rule alone on host logits [n_rows][n_vocab]: row k is session k (seeds[k], history of row k) and takes
 * draw first_draw of its stream.  A non-finite logit (NaN or +inf) is B200_EINVAL before anything runs. */
int b200_extra_sample(b200_extra_t * e, const float * logits, int n_rows, const b200_sampling_t * sp, int32_t * ids);
/* Scores sessions[k]'s tokens (counts[k] >= 2 ids, grouped by session in list order): feeds tokens 0..counts[k]-2 at the
 * session's own positions, and writes nll[j] = -log p(token j+1 | context, tokens 0..j) in float64, grouped by session
 * (sum of counts[k]-1 values).  Afterwards each session's n_past is old + counts[k] - 1 on every slice.
 *   - p is the client's perplexity arithmetic (cli_api/common.py:129-139): softmax of the row's logits in float64,
 *     m = max x, e_i = exp(x_i - m), S = sum e_i in a fixed order, nll = -log(e_t / S).  A row holding a NaN or +inf
 *     logit, or all -inf, gives NaN; a target whose e_t underflows gives +inf (the call still succeeds).
 *   - Each session's fed tokens run as one segment of one mixed pass in exact mode; sessions are packed whole, in list
 *     order, into passes of at most n_ctx rows.  So each session's logits equal one b200_session_forward of its fed
 *     tokens (fast prefill off) whatever else the call holds, and its NLLs are bit-identical alone, in a batch, or
 *     packed differently.
 *   - The host uploads the ids once, synchronises once, and reads back only nll.
 *   - Locking, slice checks and all-or-nothing errors are as b200_generate_greedy: B200_EINVAL for what it refuses
 *     (except n_steps), a count < 2 or a null nll; B200_ECONTEXT for n_past + counts[k] - 1 > n_ctx on some slice. */
int b200_score(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
               const int * counts, int n_seq, const int32_t * tokens, double * nll);
/* k_nll_rows on host logits [n_rows][n_vocab]: the kernel's test door, as b200_extra_sample is k_sample_rows'.
 * nll[k] as b200_score computes it for row k and target targets[k]; a target outside [0, n_vocab) is B200_EINVAL. */
int b200_extra_nll(b200_extra_t * e, const float * logits, int n_rows, const int32_t * targets, double * nll);

/* ---- llama.cpp's windowed perplexity (examples/perplexity/perplexity.cpp:29-117, 130) -----------------------------------
 * tokens (n_tokens ids, the text tokenized with BOS) are cut into n_chunk = n_tokens / n_ctx windows; a trailing partial
 * window is dropped, and fewer than n_ctx ids give zero windows (not an error).  n_batch is first cut to min(n_batch, n_ctx)
 * (the program's command line also caps -b at 512, examples/common.cpp:263; this call takes any n_batch).
 * Window i is tokens[i*n_ctx, (i+1)*n_ctx) with its id 0 replaced by BOS (1); it runs from n_past 0 in segments of n_batch
 * rows at positions 0, n_batch, ... (the last one may be shorter), and rows j in [first, n_ctx - 1), first =
 * min(512, n_ctx / 2), are scored against tokens[i*n_ctx + j + 1]:
 *     terms[i][j - first] = -logf(prob),  prob = (float)(e_t / S),  e_k = expf(x_k - m) (the subtraction in float),
 *     m = max x,  S = sum of the e_k in double, strictly in index order 0 .. n_vocab-1.
 * expf / logf are the double functions rounded to float: (float) exp((double) v), (float) log((double) p).  glibc's
 * expf / logf, which perplexity.cpp calls, differ from these only at float rounding midpoints.  A row with a NaN or +inf
 * logit, or all -inf, gives NaN; a prob that underflows to 0 gives +inf.  Summing the terms window by window, row by row,
 * in double gives the running perplexity perplexity.cpp prints after each window, exp(nll / count).
 *   - Windows run in waves of W = min(n_sessions, pass rows / n_batch), pass rows being the smallest slice n_ctx; window
 *     w of a wave uses sessions[w].  A wave takes ceil(n_ctx / n_batch) mixed passes, pass p carrying segment p of every
 *     window in it, so each window's rows equal b200_session_forward per segment on that window alone.  The lm_head and
 *     the term kernel run only on scored rows.
 *   - fast = 1 runs the passes' matmuls on the tensor-core prefill where a slice's format has it (Q4_0, Q8_0); other
 *     formats ignore it.  fast = 0: every row is exact.
 *   - The ids go up once (BOS already in place), the host synchronises once and reads back only terms
 *     [n_chunk][n_ctx - 1 - first].  The listed sessions are cleared first and left at n_past 0 on every slice.
 *   - Locking, slice checks and all-or-nothing errors are as b200_score: B200_EINVAL for n_ctx < 2, n_batch < 1, a
 *     session listed twice or out of range, an id outside [0, n_vocab) or a null argument; B200_ECONTEXT when n_ctx is
 *     larger than some slice's n_ctx. */
int b200_perplexity_windows(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, const int * sessions,
                            int n_sessions, const int32_t * tokens, int n_tokens, int n_ctx, int n_batch, int fast,
                            float * terms);
/* The term kernel on host logits [n_rows][n_vocab]: terms[k] as b200_perplexity_windows computes it for row k and target
 * targets[k]; a target outside [0, n_vocab) is B200_EINVAL. */
int b200_extra_ppl_terms(b200_extra_t * e, const float * logits, int n_rows, const int32_t * targets, float * terms);

/* ---- log-probabilities of generated ids ("logprobs") ------------------------------------------------------------------
 * For the logits row x (n_vocab floats) that a step drew id t from:
 *   - the distribution is the model's raw one, softmax(x) in float64: before temperature, repeat penalty and top-k/top-p,
 *     so the same whatever the sampler's settings (the sampling distribution's probabilities are not reported);
 *   - lp = log(e_t / S) with m = max x, e_i = exp((double) x_i - m) and S summed in b200_score's fixed order; the device
 *     takes m and S from the code k_nll_rows uses, so lp == -nll bit for bit, nll being b200_extra_nll of the same row and
 *     target.  An e_t that underflows gives -inf;
 *   - top-n: the n_top ids with the largest x, equal x lower id first (so in greedy mode top_ids[0] == t), each with its
 *     own log(e_i / S) from the same m and S.  0 <= n_top <= min(20, n_vocab);
 *   - a row with no distribution (a NaN or +inf logit, or all -inf) gives lp and top_lp NaN and top_ids -1; lp of an id -1
 *     (a sampled row whose scaled logits overflow) is NaN.  The id is what the call without log-probabilities gives.
 * Log-probabilities never feed back into the draw, so asking for them changes no id, and a call or stream session that asks
 * for none launches nothing extra.  Each of these calls is all-or-nothing on its arguments: B200_EINVAL, with no position
 * moved, for n_top out of range, a null lp, or a null top_ids or top_lp when n_top > 0. */
typedef struct b200_logprobs {
    int32_t  n_top;      /* 0..min(20, n_vocab): alternatives per id (0: only the drawn id's lp) */
    double * lp;         /* [n_steps][n_seq], the ids' layout */
    int32_t * top_ids;   /* [n_steps][n_seq][n_top]; may be NULL when n_top == 0 */
    double * top_lp;     /* same shape */
} b200_logprobs_t;
/* b200_generate_sample (sp NULL: b200_generate_greedy) with the log-probability of every id it writes.  The ids are those
 * calls' ids; lp row (step, k) belongs to ids[step][k].  One kernel per step after the draw, outputs on the device, copied
 * back once at the end with the ids.  A session's values are bit-identical alone, in a batch or split across calls.  Errors
 * as those calls, plus the refusals above. */
int b200_generate_lp(b200_slice_t * const * slices, int n_slices, b200_extra_t * e,
                     const int * sessions, const int * prompt_counts, int n_seq,
                     const int32_t * prompt_tokens, int n_steps, const b200_sampling_t * sp /* NULL: greedy */,
                     int32_t * ids, const b200_logprobs_t * lp);
/* b200_generate_speculative with the log-probability of every emitted id ([n_steps], n_seq = 1).  Only the emitted rows of a
 * checking pass are computed; checking rows are decode rows, bit-identical to single-token steps, so the values equal
 * b200_generate_lp's for this session alone bit for bit, whatever the draft. */
int b200_generate_speculative_lp(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int session,
                                 b200_slice_t * const * draft, int n_draft_slices, b200_extra_t * draft_e, int draft_session,
                                 const int32_t * prompt, int n_prompt, int n_steps, int n_draft,
                                 const b200_sampling_t * sp /* NULL: greedy */, int32_t * ids, b200_spec_stats_t * stats,
                                 const b200_logprobs_t * lp);
/* k_logprob_rows on host logits [n_rows][n_vocab] for ids[k] (in [0, n_vocab), else B200_EINVAL): the kernel's test door.
 * lp [n_rows], top_ids / top_lp [n_rows][n_top]. */
int b200_extra_logprobs(b200_extra_t * e, const float * logits, int n_rows, const int32_t * ids, int n_top,
                        double * lp, int32_t * top_ids, double * top_lp);

/* ---- classifier-free guidance (llama.cpp main's --cfg-negative-prompt, --cfg-scale, --cfg-smooth-factor) ---------------
 * Each generating session k has a guidance session fed a negative prompt, then the same ids session k draws.  Before each
 * draw, with b session k's logits and g its guidance session's (llama_sample_classifier_free_guidance, llama.cpp:2170-2225):
 *   log_softmax(v): m = max_element(v) (v_0 when v_0 is NaN, else the first largest non-NaN value), p_i = expf(v_i - m)
 *     with the subtraction in float, S = the p_i summed in float strictly in index order 0 .. n_vocab-1,
 *     v_i = logf(p_i / S) with the division in float;
 *   lb = log_softmax(b), lg = log_softmax(g), mix_i = fmaf(scale, lb_i - lg_i, lg_i), lg2 = log_softmax(mix),
 *   out_i = fmaf(smooth_factor, lg2_i, (1 - smooth_factor) * lb_i).
 * The two FMAs are those the reference build contracts; nothing else is fused.  expf / logf are the double functions
 * rounded to float; glibc's, which llama.cpp calls, are not correctly rounded everywhere, and that is the one place the
 * two can give different bits.  out replaces b as the row the draw reads:
 *   - greedy: max_element(out) with `<` (llama_sample_token_greedy): out_0 when it is NaN, else the first largest
 *     non-NaN value.  Where lb_i underflowed to -inf, smooth_factor 1 gives out_i = NaN (0 * -inf), and an index where
 *     lb and lg are both -inf makes the whole row NaN (id 0);
 *   - sampled: the Sampler of b200_generate_sample, unchanged, on out; a row holding a NaN has no distribution there;
 *   - a pair whose b or g holds a NaN or +inf, or is all -inf, has no distribution in either mode: its id is -1 and the
 *     call returns B200_EINVAL naming the first such step and session, after the loop (positions have moved).
 * Log-probabilities stay those of the raw b: guidance, like temperature, penalty and truncation, is not in them.  Guidance
 * is on only when asked for: at scale 1 the formula is not the identity bit for bit, so these calls refuse scale <= 1. */
typedef struct b200_guidance {
    const int * sessions;          /* [n_seq]: session k's guidance session */
    const int * prompt_counts;     /* [n_seq], >= 1: negative prompt lengths */
    const int32_t * prompt_tokens; /* the negative prompts, grouped in list order */
    float scale;                   /* finite, > 1 */
    float smooth_factor;           /* finite */
} b200_guidance_t;
/* b200_generate_lp's loop (sp NULL: greedy; lp NULL: no log-probabilities) over 2 * n_seq sessions: step 0 is one mixed
 * pass of every prompt and every negative prompt, each later step one pass of 2 * n_seq decode rows, guidance row k taking
 * the id session k drew.  The lm_head runs on both rows of each pair, then the guidance kernel, then the draw.
 *   - Positions: session k and its guidance session end at old + count + n_steps - 1 with their own counts, so a second
 *     call with prompt and negative prompt both [last id] (sampled: history and first_draw as b200_generate_sample)
 *     continues the run exactly.  A session's ids are the same alone, in a batch, or split across calls.
 *   - All-or-nothing: as b200_generate_lp, plus B200_EINVAL for a null g, a guidance session out of range, listed twice or
 *     equal to a listed session, a negative prompt count < 1 or id outside [0, n_vocab), scale not finite or <= 1, and
 *     smooth_factor not finite; B200_ECONTEXT when either context of a pair would overflow on some slice. */
int b200_generate_cfg(b200_slice_t * const * slices, int n_slices, b200_extra_t * e,
                      const int * sessions, const int * prompt_counts, int n_seq,
                      const int32_t * prompt_tokens, int n_steps, const b200_guidance_t * g,
                      const b200_sampling_t * sp /* NULL: greedy */, int32_t * ids, const b200_logprobs_t * lp /* NULL: none */);
/* The guidance kernel on host rows base / guidance [n_rows][n_vocab]: out [n_rows][n_vocab] as above, and greedy[k] (may
 * be NULL) the greedy id of row k (-1 for an all -inf input row, whose out is NaN).  A NaN or +inf input is B200_EINVAL
 * before anything runs, as are scale and smooth_factor b200_generate_cfg refuses. */
int b200_extra_cfg(b200_extra_t * e, const float * base, const float * guidance, int n_rows, float scale,
                   float smooth_factor, float * out, int32_t * greedy);

/* ---- generation streams: sessions join and leave between steps, ids reach the caller as they are drawn ----------------
 * A stream runs the generation loop of b200_generate_greedy / b200_generate_sample over a chain of slices on one GPU (the
 * same handle checks: contiguous layers, one device, no pipeline, the extra layers' n_embd), but open-ended:
 *   - b200_stream_add queues a session.  Its whole prompt is one segment of one mixed pass at the next step with room for
 *     it (on a stream opened with prefill_chunk 0: never split, a segment's rows depend on its length; see
 *     b200_stream_open_ex for chunks); decode rows of other sessions may share that pass.  Every later step feeds the
 *     session the id it drew last.  sp NULL: greedy (the argmax of the raw logits, first maximum
 *     wins); else sampled with sp's temperature, penalty, top_k and top_p, key seeds[0], history (history_counts[0] ids)
 *     and draw first_draw + j for its j-th id.  Greedy and sampled sessions with any settings share a stream.
 *   - A session ends after its max_tokens-th id, after the first id in stop_ids (delivered), or with id -1 when its logits
 *     have no distribution (see b200_generate_sample); the others go on.
 *   - b200_stream_read returns (session, id) pairs in production order: it blocks until at least one is available and
 *     writes at most cap; *n_out = 0 only when no session is active or queued.  The device runs up to `lookahead` steps
 *     ahead of the oldest step not yet read; ids of steps past a session's end are dropped.  Nothing synchronises per
 *     step: the draw kernel stores each id into a ring in mapped pinned memory that the host polls.
 *   - Each session's ids equal b200_generate_greedy / b200_generate_sample of that session alone, with the same prompt,
 *     settings and n_steps = its delivered count, whatever joined, ran beside it or left, at whichever step it joined.
 *   - Positions: when a session ends, is cancelled, or the stream closes, its n_past on every slice is
 *     old + n_prompt + delivered - 1 (old when nothing was delivered); delivered counts the ids b200_stream_read returned.
 *     So a later call with prompt = [last id], history = the delivered ids and first_draw = their count continues the run.
 *   - While a stream is open its handles belong to it: every other entry point on them (b200_session_n_past returns -1)
 *     fails with B200_EINVAL naming the stream, except b200_slice_launch_count, b200_session_count, b200_extra_dims,
 *     b200_extra_tokenize and b200_extra_token_text, which only read.  b200_stream_close gives them back.
 *   - One stream is driven from one thread.
 * b200_stream_open: max_rows = rows per step (<= the smallest n_ctx; <= 0: that n_ctx); lookahead <= 0: 4.  Sizes every
 *   buffer once.  B200_EINVAL for bad handles or sizes, B200_ENODEV without a device.  b200_stream_open_ex with
 *   prefill_chunk 0.
 * b200_stream_add: all-or-nothing.  B200_EINVAL: a session out of range or already in the stream, n_prompt < 1 or
 *   > max_rows (prefill_chunk 0 only), max_tokens < 1, an id outside [0, n_vocab) in prompt, history or stop_ids, bad
 *   sampling settings (as b200_generate_sample); B200_ECONTEXT: n_past + n_prompt + max_tokens - 1 > n_ctx on some
 *   slice.
 * b200_stream_cancel: ends a queued or active session now (B200_EINVAL if it is neither); ids not yet read are dropped.
 * b200_stream_close: ends every session, waits for the device and frees the stream. */
typedef struct b200_stream b200_stream_t;
int b200_stream_open(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int max_rows, int lookahead,
                     b200_stream_t ** out);
/* b200_stream_open whose prompts are fed in chunks of prefill_chunk = C ids, so a long prompt neither waits for a step
 * with room for all of it nor stalls the decoding sessions for a whole prompt pass.  C = 0 is b200_stream_open, bit for
 * bit and refusal for refusal.  B200_EINVAL for C < 0 or C > max_rows (after max_rows <= 0 became the smallest n_ctx).
 * With C > 0:
 *   - A prompt of n ids is fed as the chunks [0, C), [C, 2C), ... (the last one may be shorter), one segment each, at
 *     most one per session per step.  The boundaries count from the prompt's first id and never depend on what else is
 *     in the stream, so a session's rows are independent of its neighbours.  n_prompt > max_rows is accepted.
 *   - Each step, on the host: every session whose prompt is fully fed and that still owes ids gets one decode row; then
 *     the sessions with prompt ids left, in add order (so the partly fed ones before the queued ones), each get their
 *     next chunk while the step stays within max_rows; the first chunk that does not fit ends the step (no overtaking).
 *   - Only the session whose last chunk is in the step draws, from that chunk's last row; a non-final chunk takes no
 *     draw index and its rows skip the lm_head.  A step of non-final chunks only draws nothing: it stores a completion
 *     cell the host waits for before it reuses the step's buffers, and counts against lookahead as any step.
 *     b200_stream_read still blocks until an id is available.  It tops up the lookahead only while it holds no id, so
 *     the decode ids of steps beside a long prompt reach the caller step by step rather than in one burst.
 *   - Contract: a session with prompt P yields the ids (and log-probabilities) of b200_session_forward of each
 *     non-final chunk in order on every slice, then b200_generate_greedy / _sample / _lp with prompt = the last chunk,
 *     the same settings and n_steps = delivered; whatever joined, ran beside it or left.  If every prompt has at most C
 *     ids, the ids and positions are those of a prefill_chunk 0 stream.
 *   - The position rule is unchanged, also for a session cancelled or closed mid-prefill (back at old: the chunks still
 *     in flight write rows at or above old).  b200_stream_fork refuses a session still prefilling (it is active). */
int b200_stream_open_ex(b200_slice_t * const * slices, int n_slices, b200_extra_t * e, int max_rows, int lookahead,
                        int prefill_chunk, b200_stream_t ** out);
int b200_stream_add(b200_stream_t * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                    const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop);
int b200_stream_read(b200_stream_t * st, int32_t * sessions, int32_t * ids, int cap, int * n_out);
/* b200_stream_add with log-probabilities for the session's ids: n_top in [0, min(20, n_vocab)] alternatives each, -1 for
 * none (b200_stream_add).  Each session's (ids, lp, top) equal b200_generate_lp of it alone bit for bit.  A row that asks is
 * published after its record: the draw leaves its publish cell to a second kernel that writes the record into a mapped
 * logprob ring (sized once at b200_stream_open: regions x rows x (8 + 20 x 12) bytes), fences at system scope, and only then
 * stores the id.  Rows that do not ask are published by the draw as before. */
int b200_stream_add_lp(b200_stream_t * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                       const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop, int n_top);
/* b200_stream_add_lp (n_top -1: no log-probabilities) with classifier-free guidance (see b200_generate_cfg): session
 * guidance_session is fed neg (n_neg ids), then every id the session draws, and each draw reads the guided row.  The pair
 * belongs to the stream as a unit:
 *   - each step, a decoding pair has two decode rows, both taking the session's last id; b200_stream_stats counts both;
 *   - prefill: on a prefill_chunk 0 stream both prompts go whole into one step; with C > 0 each is cut into chunks counted
 *     from its own first id, each step takes the pair's next non-final chunk of each prompt as one unit (the fit and
 *     no-overtaking rule of b200_stream_open_ex), and a prompt at its final chunk waits until the other's final chunk goes
 *     in the same step, which draws;
 *   - contract: the ids (and log-probabilities, of the raw rows) equal b200_session_forward of each prompt's non-final
 *     chunks on its own session, then b200_generate_cfg with the two final chunks, the same settings and n_steps =
 *     delivered; whatever joined, ran beside it or left (so with C = 0, b200_generate_cfg with the whole prompts);
 *   - positions: the guidance session ends with the session, at old + n_neg + delivered - 1 (old when nothing was
 *     delivered, so also when cancelled mid-prefill);
 *   - while the pair is in the stream, naming the guidance session in b200_stream_add, _cancel or _fork is B200_EINVAL;
 *     cancelling the session ends both.
 * All-or-nothing as b200_stream_add, plus B200_EINVAL for a guidance session out of range, equal to session or already in
 * the stream, n_neg < 1, an id of neg outside [0, n_vocab), scale not finite or <= 1, smooth_factor not finite, or a pair
 * whose largest prefill step exceeds max_rows; B200_ECONTEXT when the guidance context would overflow. */
int b200_stream_add_cfg(b200_stream_t * st, int session, const int32_t * prompt, int n_prompt, int max_tokens,
                        const b200_sampling_t * sp, const int32_t * stop_ids, int n_stop, int n_top, int guidance_session,
                        const int32_t * neg, int n_neg, float scale, float smooth_factor);
/* b200_stream_read with each id's record: lp [cap], top_ids / top_lp [cap][20], entry j < the session's n_top filled, the
 * rest -1 / NaN; a session added without log-probabilities reads back lp NaN and top_ids -1.  b200_stream_read still works on
 * any stream and drops the records. */
int b200_stream_read_lp(b200_stream_t * st, int32_t * sessions, int32_t * ids, double * lp, int32_t * top_ids,
                        double * top_lp, int cap, int * n_out);
int b200_stream_cancel(b200_stream_t * st, int session);
/* b200_session_copy for sessions of an open stream, with one destination, on every slice of its chain: rows [0, n_keep)
 * of src to dst and dst's position to n_keep.  Enqueued on the stream's CUDA stream, so it runs after every step still in
 * flight for either session (steps left over from an earlier stay write only rows at or above that session's final
 * n_past, and the copy wins on any overlap); nothing synchronises.  dst's host position is n_keep at once, so a following
 * b200_stream_add(dst, suffix, ...) checks its context against n_keep and continues from there.  B200_EINVAL: either
 * session out of range, queued or active, src == dst, n_keep outside [0, n_past of src] on a slice, or slices whose
 * n_past of src differ. */
int b200_stream_fork(b200_stream_t * st, int src, int dst, int n_keep);
/* The stream's load so far: steps enqueued, the token rows they carried (decode rows and prompt ids), and the rows of
 * the largest step (never more than max_rows). */
int b200_stream_stats(b200_stream_t * st, int64_t * steps, int64_t * rows, int * most_rows);
int b200_stream_close(b200_stream_t * st);
/* llm.tokenize_prompt(path, prompt): BOS + sentencepiece-style merge (tensor_processor.cpp:1596-1714).
 * Returns the token count (may exceed cap; only cap are written) or a negative error. */
int b200_extra_tokenize(b200_extra_t * e, const char * prompt, int32_t * out, int cap);
/* llm.decode_token(path, id): pointer to the token's bytes (owned by the handle), length in *len. */
const char * b200_extra_token_text(b200_extra_t * e, int32_t id, int * len);

const char * b200_last_error(void);
const char * b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_SLICE_H */
