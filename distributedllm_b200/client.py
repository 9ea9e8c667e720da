"""Client-side orchestration of a layer-sliced model (reference: distllm/cli_api/common.py:9-154).

`DistributedLLM.generate / perplexity / propagate_tensor / clear_context` and `Sampler` keep the reference's
behaviour (including the shape (1, len) it sends and T=0 -> logits / 1e-5 "greedy" with repeat penalty).  The
extra layers (tokenizer, embeddings, lm_head) run through the `llm` module, which here keeps the extra-layers
file resident on the GPU instead of re-reading it on every call.

`LocalPipeline` is the on-box fast path: all slices of the nodes_map live on GPUs of this machine and the
activation never leaves HBM between them (one process, one slice handle per GPU)."""
from __future__ import annotations

import json
from typing import List, Sequence, Tuple

import numpy as np

from .capi import MAX_TOP, _int
from .compute_node.slices import import_llm
from .control_center import Connection


def parse_address(address: str) -> Tuple[str, int]:
    host, port = address.split(":")
    return host, int(port)


def load_one_slice(model_id, address_str, a, b) -> bool:
    conn = Connection(address=parse_address(address_str))
    status = conn.get_status()
    if status["status"] == "up":
        meta = status["metadata"]
        if (meta["model"], meta["layer_from"], meta["layer_to"]) == (model_id, a, b):
            return True
    for s in conn.list_all_slices():
        if (s["model"], s["layer_from"], s["layer_to"]) == (model_id, a, b):
            conn.load_slice(s["name"])
            return True
    return False


def get_llm(config_path, registry_path="models_registry/registry.json"):
    with open(config_path) as f:
        config = json.load(f)
    items = list(config["nodes_map"].items())
    for address_str, (a, b) in items:
        load_one_slice(config["model_id"], address_str, a, b)
    nodes = [parse_address(addr) for addr, _ in sorted(items, key=lambda t: t[1])]
    with open(registry_path) as f:
        registry = json.load(f)
    return DistributedLLM(nodes, registry[config["model_id"]]["extra_layers_file"])


def _softmax(x: np.ndarray, axis=-1) -> np.ndarray:
    x = x - x.max(axis=axis, keepdims=True)
    e = np.exp(x)
    return e / e.sum(axis=axis, keepdims=True)


def token_logprobs(logits, token, n_top: int):
    """The log-probability of `token` under the raw distribution softmax(logits) in float64, and the n_top ids of largest
    logit (equal logits: lower id first) with theirs: the host twin of the device's logprobs (include/b200_slice.h).
    -> (lp, [(id, lp), ...]).  A row with a NaN or +inf logit, or all -inf, has no distribution: lp NaN and every
    alternative (-1, NaN).  A token whose probability underflows gives -inf.  The sum runs in numpy's order, so values
    agree with the device's within ~1e-15 relative, not bit for bit."""
    x = np.asarray(logits, dtype=np.float32).reshape(-1).astype(np.float64)
    n = len(x)
    if n < 1:
        raise ValueError("logits must hold at least one value")
    token = _int("token", token, 0, n - 1)
    n_top = _int("n_top", n_top, 0, min(MAX_TOP, n))
    if np.isnan(x).any() or (x == np.inf).any() or (x == -np.inf).all():
        return float("nan"), [(-1, float("nan"))] * n_top
    with np.errstate(divide="ignore"):
        e = np.exp(x - x.max())
        S = e.sum()
        lp = lambda i: float(np.log(e[i] / S))
        top = np.lexsort((np.arange(n), -x))[:n_top]
        return lp(token), [(int(i), lp(i)) for i in top]


def ppl_terms(logits, targets) -> np.ndarray:
    """llama.cpp's perplexity term for each row of [n][n_vocab] logits (perplexity.cpp:12-26, 103-113), the host twin of
    the device's (include/b200_slice.h): m = max x, e_i = expf(x_i - m) with the subtraction in float32, S = the e_i
    summed in float64 strictly in index order (a sequential cumsum: np.sum is pairwise), prob = float32(e_t / S),
    term = -logf(prob).  expf / logf are float64 exp / log rounded to float32, as on the device; glibc's expf / logf, which
    perplexity.cpp calls, differ from them only near float midpoints.  A row with a NaN or +inf logit, or all -inf, gives
    NaN; a prob that underflows to 0 gives +inf.  -> [n] float32."""
    t = np.asarray(targets, dtype=np.int64).reshape(-1)
    x = np.asarray(logits, dtype=np.float32).reshape(len(t), -1)
    out = np.empty(len(t), np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for k, (row, tk) in enumerate(zip(x, t)):
            if np.isnan(row).any() or (row == np.inf).any() or (row == -np.inf).all():
                out[k] = np.nan
                continue
            e = np.exp((row - row.max()).astype(np.float64)).astype(np.float32)
            S = np.cumsum(e, dtype=np.float64)[-1]
            prob = np.float32(np.float64(e[tk]) / S)
            out[k] = -np.float32(np.log(np.float64(prob)))
    return out


def _exp_f32(v: np.ndarray) -> np.ndarray:
    return np.exp(v.astype(np.float64)).astype(np.float32)


def _log_f32(v: np.ndarray) -> np.ndarray:
    return np.log(v.astype(np.float64)).astype(np.float32)


def _fma_f32(a, b, c) -> np.ndarray:
    """float32 fma(a, b, c), rounded once: float64 a*b is exact, and a TwoSum plus round-to-odd keeps the float64 sum from
    rounding twice."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c64 = np.asarray(c, np.float32).astype(np.float64)
    hi = p + c64
    bb = hi - p
    lo = (p - (hi - bb)) + (c64 - bb)
    odd = (lo != 0) & ((hi.view(np.int64) & 1) == 0) & np.isfinite(hi)
    hi = np.where(odd, np.nextafter(hi, np.where(lo > 0, np.inf, -np.inf)), hi)
    return hi.astype(np.float32)


def _log_softmax_f32(v: np.ndarray, expf, logf) -> np.ndarray:
    """llama_log_softmax (llama.cpp:2170-2182) on one float32 row: m = *max_element (v_0 when it is NaN), p = expf(v - m),
    the p summed in float32 in index order (np.add.accumulate is sequential), logf(p / sum)."""
    m = v[0] if np.isnan(v[0]) else np.nanmax(v)
    p = expf(v - np.float32(m))
    S = np.add.accumulate(p, dtype=np.float32)[-1]
    return logf(p / S)


def cfg_logits(base, guidance, scale: float, smooth_factor: float, expf=_exp_f32, logf=_log_f32) -> np.ndarray:
    """llama.cpp's classifier-free guidance (llama_sample_classifier_free_guidance) for each row pair of [n][n_vocab]
    logits, the host twin of the device's (include/b200_slice.h): lb = log_softmax(base), lg = log_softmax(guidance),
    mix = fmaf(scale, lb - lg, lg), out = fmaf(sf, log_softmax(mix), (1 - sf) * lb), every step in float32 and the two
    FMAs rounded once.  expf / logf default to float64 exp / log rounded to float32, as on the device; pass libm's to get
    the reference build's bits.  -> float32 [n][n_vocab]."""
    b = np.asarray(base, np.float32)
    g = np.asarray(guidance, np.float32).reshape(b.shape)
    b2, g2 = b.reshape(-1, b.shape[-1]), g.reshape(-1, b.shape[-1])
    out = np.empty_like(b2)
    sc, sf = np.float32(scale), np.float32(smooth_factor)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
        for k in range(len(b2)):
            lb, lg = _log_softmax_f32(b2[k], expf, logf), _log_softmax_f32(g2[k], expf, logf)
            lg2 = _log_softmax_f32(_fma_f32(sc, lb - lg, lg), expf, logf)
            out[k] = _fma_f32(sf, lg2, (np.float32(1) - sf) * lb)
    return out.reshape(b.shape)


def cfg_greedy(row) -> int:
    """llama_sample_token_greedy on one row: std::max_element with `<` -- the first element when it is NaN, else the
    first largest non-NaN value."""
    row = np.asarray(row, np.float32)
    if np.isnan(row[0]):
        return 0
    return int(np.nanargmax(row))


def running_perplexity(terms) -> List[float]:
    """The values perplexity.cpp prints after each window, from terms [n_chunk][n_scored]: nll (float64) adds the terms
    window by window, row by row,
    then exp(nll / count) (perplexity.cpp:111-115)."""
    out, nll, count = [], 0.0, 0
    for row in np.asarray(terms, np.float32):
        for v in row:
            nll += float(v)
            count += 1
        out.append(float(np.exp(nll / count)) if count else float("nan"))
    return out


def windowed_perplexity_terms(tokens, n_ctx: int, n_batch: int, eval_segment) -> np.ndarray:
    """perplexity.cpp's loop (:37-113) on the host: for each whole window of n_ctx ids, with its id 0 replaced by BOS,
    eval_segment(ids, n_past) -> logits [len(ids)][n_vocab] is called segment by segment (n_past 0 starts a window), and
    the scored rows' terms are ppl_terms of those logits.  -> float32 [n_chunk][n_scored]."""
    from .capi import ppl_window_rows
    tokens = [int(t) for t in tokens]
    n_chunk, n_batch, first, n_scored = ppl_window_rows(len(tokens), n_ctx, n_batch)
    out = np.zeros((n_chunk, n_scored), np.float32)
    for i in range(n_chunk):
        start = i * n_ctx
        ids = [1] + tokens[start + 1:start + n_ctx]          # llama_token_bos()
        logits = np.concatenate([np.asarray(eval_segment(ids[j:j + n_batch], j), np.float32).reshape(len(ids[j:j + n_batch]), -1)
                                 for j in range(0, n_ctx, n_batch)])
        if n_scored:
            out[i] = ppl_terms(logits[first:n_ctx - 1], tokens[start + first + 1:start + n_ctx])
    return out


class Sampler:
    """The reference's sampler, plus llama.cpp's top-k and top-p truncation (off when both are None, which runs the
    reference's arithmetic unchanged).  Truncation ranks the ids by the scaled logits y descending (equal y: lower id
    first), keeps the first top_k of them (0 or None: all), then within those keeps an id iff the probability ranked
    strictly before it is < top_p times their total (0, None or >= 1: no cut; the top id is always kept), and draws from
    the kept probabilities with the same single random() and the same id-order rule."""

    def __init__(self, temperature=0.7, repeat_penalty=1.1, rng=None, top_k=None, top_p=None):
        self.T = temperature
        self.penalty = repeat_penalty
        self.previous_ids: List[int] = []
        self.eps = 10 ** (-5)
        self.rng = rng or np.random
        self.top_k = top_k
        self.top_p = top_p

    def __call__(self, logits) -> int:
        logits = np.array(logits)
        ids = np.arange(len(logits))
        seen = np.isin(ids, self.previous_ids)
        logits = logits / ((seen * self.penalty + ~seen) * (self.T + self.eps))
        if self.top_k is None and self.top_p is None:
            token_id = int(self.rng.choice(ids, p=_softmax(logits)))
        else:
            p = _softmax(logits)
            order = np.lexsort((ids, -logits))                  # y descending, lower id first
            K = order[:self.top_k] if self.top_k else order
            keep = np.zeros(len(ids), bool)
            keep[K] = True
            if self.top_p and self.top_p < 1:
                pk = p[K]
                before = np.concatenate(([0.0], np.cumsum(pk)[:-1]))
                keep[K[before >= self.top_p * pk.sum()]] = False
            p = np.where(keep, p, 0.0)
            token_id = int(self.rng.choice(ids, p=p / p.sum()))
        self.previous_ids.append(token_id)
        return token_id


class DistributedLLM:
    def __init__(self, addresses: Sequence[Tuple[str, int]], extra_layers_path: str, wire: str = "list"):
        """wire: "list"  -- the reference's per-node star of float lists (common.py:148-154);
                 "bytes" -- same star, tensors as one binary field;
                 "chain" -- binary, and the nodes pass the activation along themselves: one client round trip per step."""
        if wire not in ("list", "bytes", "chain"):
            raise ValueError("wire must be list, bytes or chain")
        self.addresses = list(addresses)
        self.extra_layers_path = extra_layers_path
        self.wire = wire
        self.llm = import_llm()

    def generate(self, prompt, max_steps=200, temperature=0.0, repeat_penalty=1.1, rng=None, top_k=None, top_p=None,
                 logprobs=None):
        """rng: the Sampler's random generator (default numpy's global one, as the reference);
        numpy.random.Generator(numpy.random.Philox(key=seed)) gives LocalPipeline.generate's ids for that seed.
        top_k / top_p: the Sampler's truncation (None: off).  logprobs = n_top (0..20): yield (text, lp, [(id, lp), ...])
        instead of text, from token_logprobs on each step's logits."""
        if logprobs is not None:
            logprobs = _int("logprobs", logprobs, 0, MAX_TOP)
        self.clear_context()
        extra = self.extra_layers_path
        tokens = self.llm.tokenize_prompt(extra, prompt)
        sampler = Sampler(temperature, repeat_penalty, rng=rng, top_k=top_k, top_p=top_p)
        for _ in range(max_steps):
            emb = self.propagate_tensor(self.llm.prepare_embeddings(extra, tokens))
            logits = self.llm.get_logits(extra, emb, False)
            token_id = sampler(logits)
            tokens = [token_id]
            text = self.llm.decode_token(extra, token_id)
            if logprobs is None:
                yield text
            else:
                yield (text, *token_logprobs(logits, token_id, logprobs))

    def generate_greedy(self, prompt, max_steps=200) -> List[int]:
        """Pure argmax decoding through llm.get_next_token (tensor_processor.cpp:1894-1908): the parity path."""
        self.clear_context()
        extra = self.extra_layers_path
        tokens = self.llm.tokenize_prompt(extra, prompt)
        out = []
        for _ in range(max_steps):
            emb = self.propagate_tensor(self.llm.prepare_embeddings(extra, tokens))
            token_id = self.llm.get_next_token(extra, emb)
            out.append(token_id)
            tokens = [token_id]
        return out

    def perplexity(self, text) -> float:
        self.clear_context()
        extra = self.extra_layers_path
        tokens = self.llm.tokenize_prompt(extra, text)
        emb = self.propagate_tensor(self.llm.prepare_embeddings(extra, tokens[:-1]))
        n = len(tokens) - 1
        logits = np.array(self.llm.get_logits(extra, emb, True)).reshape(n, -1)
        p = _softmax(logits, axis=1)[np.arange(n), tokens[1:]]
        return float(np.exp(-np.log(p).sum() / n))

    def perplexity_windows(self, text, n_ctx: int = 512, n_batch: int = 512) -> List[float]:
        """llama.cpp's windowed perplexity through the nodes: each window starts from cleared contexts and is fed segment
        by segment, with get_logits(all) after each; the terms are ppl_terms.  -> the running perplexity after each
        window, as perplexity.cpp prints it."""
        extra = self.extra_layers_path
        tokens = self.llm.tokenize_prompt(extra, text)

        def eval_segment(ids, n_past):
            if n_past == 0:
                self.clear_context()
            emb = self.propagate_tensor(self.llm.prepare_embeddings(extra, ids))
            return np.array(self.llm.get_logits(extra, emb, True), np.float32).reshape(len(ids), -1)

        return running_perplexity(windowed_perplexity_terms(tokens, n_ctx, n_batch, eval_segment))

    def clear_context(self):
        for address in self.addresses:
            Connection(address).clear_context()

    def propagate_tensor(self, embeddings):
        shape = (1, len(embeddings))
        if self.wire == "list":
            for address in self.addresses:
                embeddings = Connection(address).propagate_forward(embeddings, shape)["values"]
            return embeddings
        x = np.asarray(embeddings, dtype=np.float32)
        if self.wire == "bytes":
            for address in self.addresses:
                x = Connection(address).propagate_forward_bytes(x, shape)
        else:
            route = ["%s:%d" % (h, p) for h, p in self.addresses[1:]]
            x = Connection(self.addresses[0]).propagate_forward_bytes(x, shape, route)
        return x.tolist()


# llama_token_eos(): the end-of-sequence id of the LLaMA vocabulary (LocalPipeline.generate(stop_at_eos=True))
EOS_ID = 2


class LocalPipeline:
    """All slices of a nodes_map on the GPUs of THIS box: slice i on device i, activations chained device to
    device (peer copy) -- the single-process equivalent of the NCCL pipeline bench.py runs with one rank per GPU."""

    def __init__(self, slice_paths: Sequence[str], devices: Sequence[int] = None, n_ctx: int = 0, n_sessions: int = 1,
                 lora: str = None, lora_base: str = None):
        """n_sessions: KV-cache sessions per slice (perplexity_windows runs up to that many windows per pass).
        lora: one adapter file applied to every slice (capi.Slice); each slice takes the adapter's tensors for its own
        layers.  lora_base: the F16 / F32 base as one slice file covering every slice's layers, or one file per slice."""
        from . import capi
        self.capi = capi
        devices = list(devices) if devices is not None else list(range(len(slice_paths)))
        if isinstance(lora_base, str) or lora_base is None:
            lora_base = [lora_base] * len(slice_paths)
        self.slices = [capi.Slice(p, d, n_ctx, n_sessions=n_sessions, lora=lora, lora_base=b)
                       for p, d, b in zip(slice_paths, devices, lora_base)]
        self.slices.sort(key=lambda s: s.info.first_layer)
        self._extra = None

    def _device_extra(self, extra_path: str, what: str):
        """The extra layers on the slices' one GPU, loaded once per path."""
        devices = sorted({s.info.device for s in self.slices})
        if len(devices) != 1:
            raise self.capi.B200Error(1, "%s on the device needs every slice on one GPU; the slices are on "
                                         "devices %s" % (what, ", ".join(map(str, devices))))
        if self._extra is None or self._extra[0] != extra_path:
            if self._extra is not None:
                self._extra[1].close()
            self._extra = (extra_path, self.capi.Extra(extra_path, devices[0]))
        return self._extra[1]

    def _guidance(self, extra, cfg_negative_prompt, cfg_scale: float, cfg_smooth_factor: float):
        """llama.cpp main's --cfg-negative-prompt / --cfg-scale / --cfg-smooth-factor as capi's guidance= argument:
        None when guidance is off (no negative prompt, or cfg_scale <= 1, as main), else session 1 fed the negative prompt,
        tokenized as the prompt is."""
        if cfg_negative_prompt is None or not cfg_scale > 1:
            return None
        if self.slices[0].n_sessions < 2:
            raise ValueError("classifier-free guidance runs the negative prompt in session 1: load the slices with "
                             "n_sessions >= 2 (they have %d)" % self.slices[0].n_sessions)
        return ([1], [extra.tokenize(cfg_negative_prompt)], float(cfg_scale), float(cfg_smooth_factor))

    def generate_greedy(self, extra_path: str, prompt: str, max_steps: int = 200, logprobs: int = None,
                        cfg_negative_prompt: str = None, cfg_scale: float = 1.0, cfg_smooth_factor: float = 1.0) -> list:
        """DistributedLLM.generate_greedy on this box: clear the contexts, tokenize, then max_steps argmax steps, all on
        the GPU with no host round trip between tokens (capi.generate_greedy).  Needs every slice on one device.
        logprobs = n_top (0..20): a list of (id, lp, [(id, lp), ...]) instead of ids.  cfg_negative_prompt with
        cfg_scale > 1: llama.cpp main's classifier-free guidance (capi.generate_greedy's guidance=), the negative prompt in
        session 1; the log-probabilities stay those of the unguided logits."""
        extra = self._device_extra(extra_path, "greedy generation")
        if logprobs is not None:
            logprobs = _int("logprobs", logprobs, 0, MAX_TOP)
        guidance = self._guidance(extra, cfg_negative_prompt, cfg_scale, cfg_smooth_factor)
        self.clear_context()
        if guidance is not None:
            for sl in self.slices:
                sl.session_clear(1)
        tokens = extra.tokenize(prompt)
        if max_steps < 1:
            return []
        if guidance is not None:
            out = self.capi.generate_greedy(self.slices, extra, [0], [tokens], max_steps, logprobs=logprobs, guidance=guidance)
            if logprobs is None:
                return out[:, 0].tolist()
            ids, lp, ti, tl = out
            return _with_logprobs(ids[:, 0], lp[:, 0], ti[:, 0], tl[:, 0])
        if logprobs is None:
            return self.capi.generate_greedy(self.slices, extra, [0], [tokens], max_steps)[:, 0].tolist()
        ids, lp, ti, tl = self.capi.generate_greedy(self.slices, extra, [0], [tokens], max_steps, logprobs=logprobs)
        return _with_logprobs(ids[:, 0], lp[:, 0], ti[:, 0], tl[:, 0])

    def generate(self, extra_path: str, prompt: str, max_steps: int = 200, temperature: float = 0.0,
                 repeat_penalty: float = 1.1, seed: int = None, stop_at_eos: bool = False, top_k: int = None,
                 top_p: float = None, logprobs: int = None, cfg_negative_prompt: str = None, cfg_scale: float = 1.0,
                 cfg_smooth_factor: float = 1.0):
        """DistributedLLM.generate on this box: clear the contexts, tokenize, then up to max_steps steps of the client's
        Sampler, all on the GPU with no host round trip between tokens (a one-session capi.Stream).  Yields each token
        string as soon as its id is drawn; leaving the loop early cancels the steps that remain, and the slices' n_past
        is then len(prompt tokens) + (strings yielded) - 1.  The draws come from numpy.random.Philox(key=seed), so
        DistributedLLM.generate(..., rng=numpy.random.Generator(numpy.random.Philox(key=seed))) yields the same strings.
        seed=None draws a key from numpy's global generator, so unseeded runs vary as the reference's do.
        stop_at_eos=True ends the run after the end-of-sequence id (EOS_ID, yielded); the default runs max_steps steps,
        as the reference does.  top_k / top_p truncate each draw as client.Sampler does (None: off).  logprobs = n_top
        (0..20): yield (text, lp, [(id, lp), ...]) as DistributedLLM.generate does, from the stream's records.  Needs
        every slice on one device.
        cfg_negative_prompt with cfg_scale > 1: llama.cpp main's classifier-free guidance, the Sampler drawing from the
        guided rows (capi.Stream.add's guidance=, the negative prompt in session 1, which ends with session 0)."""
        extra = self._device_extra(extra_path, "sampled generation")
        if logprobs is not None:
            logprobs = _int("logprobs", logprobs, 0, MAX_TOP)
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 64, dtype=np.uint64))
        guidance = self._guidance(extra, cfg_negative_prompt, cfg_scale, cfg_smooth_factor)
        self.clear_context()
        if guidance is not None:
            for sl in self.slices:
                sl.session_clear(1)
        tokens = extra.tokenize(prompt)
        if max_steps < 1:
            return
        with self.capi.Stream(self.slices, extra) as st:
            st.add(0, tokens, max_steps, temperature, repeat_penalty, seed, stop_ids=[EOS_ID] if stop_at_eos else (),
                   top_k=top_k or 0, top_p=top_p or 0.0, logprobs=logprobs,
                   guidance=None if guidance is None else (1, guidance[1][0], guidance[2], guidance[3]))
            records = iter(st) if logprobs is None else _read_records(st)
            for j, rec in enumerate(records):
                token_id = rec[1]
                if token_id < 0:
                    raise self.capi.B200Error(1, "step %d: the logits hold a NaN or +inf, are all -inf or overflow "
                                                 "float64 once scaled, so they have no distribution" % j)
                if logprobs is None:
                    yield extra.token_text(token_id)
                else:
                    yield extra.token_text(token_id), rec[2], rec[3]

    def generate_speculative(self, extra_path: str, prompt: str, draft: "LocalPipeline", draft_extra_path: str,
                             max_steps: int = 200, n_draft: int = 4, temperature: float = 0.0, repeat_penalty: float = 1.1,
                             seed: int = None, top_k: int = None, top_p: float = None, logprobs: int = None) -> list:
        """Speculative decoding on this box (capi.generate_speculative): clear both pipelines' contexts, tokenize with the
        target's extra layers, then max_steps ids, the draft pipeline proposing n_draft ids per target pass.  The ids do
        not depend on the draft: at temperature 0 they are generate_greedy's; otherwise the ids behind the strings
        generate(..., seed=seed, stop_at_eos=False) yields.  Needs every slice of both pipelines on one device.
        logprobs = n_top (0..20): a list of (id, lp, [(id, lp), ...]) instead of ids, equal to the plain loop's."""
        extra = self._device_extra(extra_path, "speculative generation")
        if logprobs is not None:
            logprobs = _int("logprobs", logprobs, 0, MAX_TOP)
        dextra = draft._device_extra(draft_extra_path, "speculative generation")
        if temperature and seed is None:
            seed = int(np.random.randint(0, 2 ** 64, dtype=np.uint64))
        self.clear_context()
        draft.clear_context()
        tokens = extra.tokenize(prompt)
        if max_steps < 1:
            return []
        out, _ = self.capi.generate_speculative(self.slices, extra, 0, draft.slices, dextra, 0, tokens, max_steps, n_draft,
                                                temperature=temperature if temperature else None,
                                                repeat_penalty=repeat_penalty, seed=seed, top_k=top_k or 0,
                                                top_p=top_p or 0.0, logprobs=logprobs)
        return out.tolist() if logprobs is None else _with_logprobs(*out)

    def perplexity(self, extra_path: str, text: str) -> float:
        """DistributedLLM.perplexity on this box: clear the contexts, tokenize, then score the text on the GPU
        (capi.score: one pass, lm_head and softmax on the device, only the per-token NLLs come back).  The NLLs are
        summed in the reference's order (one `nll -= log p` per token, cli_api/common.py:136-139).  Needs every slice
        on one device."""
        extra = self._device_extra(extra_path, "scoring")
        self.clear_context()
        tokens = extra.tokenize(text)
        n = len(tokens) - 1
        nll = 0.0
        for v in self.capi.score(self.slices, extra, [0], [tokens])[0]:
            nll += v
        return float(np.exp(nll / n))

    def perplexity_windows(self, extra_path: str, text: str, n_ctx: int = 512, n_batch: int = 512, sessions=None,
                           fast: bool = False) -> List[float]:
        """llama.cpp's `perplexity` on this box (capi.perplexity_windows): tokenize with BOS, cut into windows of n_ctx
        ids, evaluate each from an empty context in segments of n_batch rows, score the second half of each window on
        the device.  -> the running perplexity after each window, as perplexity.cpp prints it (nll summed in float64 in
        its order).  sessions: the sessions that windows run in side by side (default: every session of the slices, so
        load them with n_sessions > 1 for several windows per pass); they are left at n_past 0.  fast: the
        tensor-core prefill on Q4_0 / Q8_0 slices.  Needs every slice on one device."""
        extra = self._device_extra(extra_path, "windowed perplexity")
        if sessions is None:
            sessions = list(range(min(s.n_sessions for s in self.slices)))
        tokens = extra.tokenize(text)
        terms = self.capi.perplexity_windows(self.slices, extra, sessions, tokens, n_ctx, n_batch, fast=fast)
        return running_perplexity(terms)

    def propagate_tensor(self, embeddings) -> np.ndarray:
        x = np.ascontiguousarray(embeddings, dtype=np.float32)
        for s in self.slices:
            x = s.forward(x)
        return x

    def clear_context(self):
        for s in self.slices:
            s.clear_context()

    def close(self):
        if self._extra is not None:
            self._extra[1].close()
            self._extra = None
        for s in self.slices:
            s.close()


def _with_logprobs(ids, lp, top_ids, top_lp) -> list:
    """Arrays of a logprobs call for one session -> [(id, lp, [(id, lp), ...]), ...]."""
    return [(int(t), float(v), [(int(a), float(b)) for a, b in zip(ti, tl)]) for t, v, ti, tl in zip(ids, lp, top_ids, top_lp)]


def _read_records(st):
    """A stream's (session, id, lp, alternatives) records, one at a time, until no session is left."""
    while True:
        recs = st.read_logprobs(1)
        if not recs:
            return
        yield recs[0]
