"""GPU: the vocabulary-sized kernels at vocabulary sizes that are not a multiple of 32 -- where the lm_head's last row
group, the penalty bitmaps' last word and the sampler's last thread chunk are only partly filled.

Real GGJT files have such sizes: fine-tunes that add a pad token have 32001 ids, Chinese-LLaMA 49953.  Each test asserts
that it reached the ragged tail (ids in the last bitmap word were computed, drawn, scored), not only that it ran.

  a. lm_head and embedding: Extra.logits / Extra.embed against the reference's digests (tests/golden/
     ref_digests_vocab.json), every output type, bit for bit; each row equal to that row computed alone.
  b. argmax: output.weight edited so that the maximum lands at V - 1, at 32*floor(V/32), or ties an early id with V - 1;
     Extra.next_token and generate_greedy against the first-maximum rule on the C restatement's logits.
  c. sampler and truncation: Extra.sample against the host twin (tests/trunc_ref.py) under its ambiguity rule, and the
     device-only properties (a cut that drops nothing changes no bit; a row's id does not depend on its batch position).
  d. NLL: Extra.nll against tests/score_ref.py.
  e. the device loops at V = 32001: generate_greedy, generate_sample with top_k 40 / top_p 0.95, score and a Stream,
     against the host loop and each session alone."""
import json
import os
import sys

import numpy as np
import pytest

import edge_cases as ec
import sample_ref
import score_ref
import trunc_ref
from distributedllm_b200 import ggjt
from test_gpu_sample import _rows
from test_gpu_truncated_sample import _edge_rows, _host_loop as _sample_host_loop, _settings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import gen_golden_vocab as vocab_ref  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(HERE, "golden", "ref_digests_vocab.json")))
SAMPLE_VOCABS = (1024, 1025, 1031, 32001, 32767, 32768, 49953)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _word(n_vocab: int) -> int:
    """The first id of the last 32-id penalty-bitmap word."""
    return (n_vocab - 1) // 32 * 32


# --------------------------------------------------------------------------- a. lm_head and embedding
@pytest.mark.parametrize("name", sorted(CASES))
def test_lm_head_and_embedding_match_the_reference(tmp_path, name):
    from distributedllm_b200 import capi
    case = CASES[name]
    v = case["n_vocab"]
    path = str(tmp_path / "extra.bin")
    vocab_ref.write_extra(path, case)
    assert vocab_ref.file_sha256(path) == case["file_sha256"], "the writer changed: regenerate the fixture"
    extra = capi.Extra(path, 0)
    assert (extra.n_vocab, extra.n_embd) == (v, case["n_embd"])
    for n, want in zip(case["rows"], case["logits"]):
        x = vocab_ref.hidden(case, n)
        y = extra.logits(x)
        got = [vocab_ref.digest(r) for r in y]
        if got != want:
            port = ec.port_logits(path, x)
            bad = [(i, int((_bits(y[i]) != _bits(port[i])).sum()), np.flatnonzero(_bits(y[i]) != _bits(port[i]))[:5].tolist())
                   for i in range(n) if got[i] != want[i]]
            pytest.fail("%s, %d rows: rows (row, ids differing from the restatement, first ids) %s" % (name, n, bad))
        assert np.any(y[:, vocab_ref.tail_ids(v)[3]:] != 0), (name, n)        # the tail rows were computed
        for i in range(n):
            assert (_bits(extra.logits(x[i:i + 1])[0]) == _bits(y[i])).all(), (name, n, i)
    ids = case["embed_ids"]
    emb = extra.embed(ids)
    port = ec.dequant_rows(ggjt.read_file(path, sliced=True), "tok_embeddings.weight", ids)
    assert (_bits(emb) == _bits(port)).all(), name
    if case["embed"] is not None:
        assert [vocab_ref.digest(r) for r in emb] == case["embed"], name
    extra.close()


# --------------------------------------------------------------------------- b. argmax
_SCALE_OFFSETS = {ggjt.T_Q4_0: (0,), ggjt.T_Q4_1: (0, 2), ggjt.T_Q5_0: (0,), ggjt.T_Q5_1: (0, 2), ggjt.T_Q8_0: (0,),
                  ggjt.T_Q6_K: (208,)}


def _edit_output(src: str, dst: str, copies: dict, factor: float) -> None:
    """Write dst: src with output.weight row r replaced by row copies[r] with every block scale (and minimum) times
    factor.  A power of two scales every product and sum exactly, so logit(r) = factor * logit(copies[r])."""
    f = ggjt.read_file(src, sliced=True)

    def gen():
        for name, t in f.tensors.items():
            raw = f.read_raw(name)
            if name == "output.weight":
                w = ec._blocks(raw, t.ttype, t.ne)
                for r, a in copies.items():
                    if t.ttype == ggjt.T_F16:
                        w[r] = (w[a].astype(np.float32) * np.float32(factor)).astype(np.float16)
                        continue
                    w[r] = w[a]
                    sel = np.zeros(w.shape[:2], bool)
                    sel[r] = True
                    for o in _SCALE_OFFSETS[t.ttype]:
                        s = ec._get_f16(w, o)[sel].astype(np.float32) * np.float32(factor)
                        ec._set_f16(w, o, sel, s.astype(np.float16).view(np.uint16))
                raw = np.ascontiguousarray(w).tobytes()
            yield name, t.ttype, t.ne, raw

    ggjt.write_file(dst, f.hparams, f.vocab, list(gen()))


def _greedy_host(slices, extra, session, prompt, n_steps):
    """The client's greedy loop through the host with the logits on the host: Extra.logits, then numpy's first maximum."""
    ids, toks = [], list(prompt)
    for _ in range(n_steps):
        x = extra.embed(toks)
        for s in slices:
            x = s.session_forward(session, x)
        ids.append(int(np.argmax(extra.logits(x)[-1])))
        toks = [ids[-1]]
    return ids


@pytest.mark.parametrize("n_vocab,out", [(1031, ggjt.T_Q4_0), (32001, ggjt.T_Q4_0), (49953, ggjt.T_Q4_0),
                                         (32001, ggjt.T_Q6_K), (1031, ggjt.T_F16)])
def test_argmax_at_the_vocabulary_tail(tmp_path, n_vocab, out):
    """The maximum at V - 1, at the first id of the last bitmap word, and tied between an early id and V - 1 (the early
    id wins): Extra.next_token (k_argmax_first) and generate_greedy (k_argmax_rows) against the first-maximum rule."""
    from distributedllm_b200 import capi
    sh = ggjt.ModelShape(n_vocab, 256, 256, 4, 2)
    base = str(tmp_path / "extra.bin")
    if out == ggjt.T_Q6_K:
        ggjt.write_kquant_extra(base, sh, "q4_K_M", seed=21)
    else:
        ggjt.write_synth_extra(base, sh, out, seed=21)
    paths = [str(tmp_path / "a.bin"), str(tmp_path / "b.bin")]
    ggjt.write_synth_slice(paths[0], sh, 0, 0, ggjt.T_Q4_0, seed=21)
    ggjt.write_synth_slice(paths[1], sh, 1, 1, ggjt.T_Q4_0, seed=21)
    gpu = [capi.Slice(p, 0, 64, n_sessions=4) for p in paths]
    twin = [capi.Slice(p, 0, 64, n_sessions=4) for p in paths]
    extra = capi.Extra(base, 0)
    rng = np.random.default_rng(n_vocab)
    prompts = [rng.integers(0, n_vocab, n).tolist() for n in (3, 1, 6, 2)]
    x = extra.embed(prompts[0])                    # session 0's last hidden state: the row the edits aim at
    for s in twin:
        x = s.session_forward(0, x)
    for s in twin:
        s.session_clear(-1)
    h = np.concatenate([x[-1:], rng.standard_normal((3, sh.n_embd), dtype=np.float32)])
    extra.close()
    l0 = ec.port_logits(base, h)
    a = int(np.argmax(l0[0]))
    assert l0[0, a] > 0
    w, early = _word(n_vocab), 3 if a != 3 else 4
    variants = {"last": ({n_vocab - 1: a}, n_vocab - 1), "word": ({w: a}, w),
                "tie": ({early: a, n_vocab - 1: a}, early)}
    for tag, (copies, want) in variants.items():
        path = str(tmp_path / ("extra_%s.bin" % tag))
        _edit_output(base, path, copies, 2.0)
        port = ec.port_logits(path, h)
        for r in copies:
            assert port[0, r] == 2 * l0[0, a], (tag, r)
        assert int(np.argmax(port[0])) == want, tag
        extra = capi.Extra(path, 0)
        assert (_bits(extra.logits(h)) == _bits(port)).all(), tag
        assert extra.next_token(h[:1]) == want, tag
        for i in range(1, len(h)):
            assert extra.next_token(h[:i + 1]) == int(np.argmax(port[i])), (tag, i)
        ids = capi.generate_greedy(gpu, extra, [0, 1, 2, 3], prompts, 3)
        assert ids[0, 0] == want, tag
        for k in range(4):
            assert _greedy_host(twin, extra, k, prompts[k], 3) == ids[:, k].tolist(), (tag, k)
        for s in gpu + twin:
            s.session_clear(-1)
        extra.close()
    for s in gpu + twin:
        s.close()


# --------------------------------------------------------------------------- c. sampler and truncation
def _sample_extra(tmp_path, n_vocab):
    from distributedllm_b200 import capi
    path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(path, ggjt.ModelShape(n_vocab, 256, 256, 4, 1), ggjt.T_Q4_0, seed=62)
    extra = capi.Extra(path, 0)
    assert extra.n_vocab == n_vocab
    return extra


def _tail_rows(rng, n):
    """-> (rows, histories): mass and ties in the last bitmap word and the last thread chunk of sample_row."""
    w = _word(n)
    chunk = (n + 1023) // 1024
    last_chunk = (n - 1) // chunk * chunk                    # first id of the last thread's chunk
    rows, hist = [], []
    r = rng.standard_normal(n)
    r[n - 1] += 9.0
    rows.append(r); hist.append([])                         # the mass at V - 1
    r = np.full(n, -np.inf)
    r[w:] = rng.standard_normal(n - w)
    rows.append(r); hist.append([n - 1])                    # only the last word is finite, V - 1 penalised
    r = np.full(n, -3.0)
    r[w:] = 2.0
    r[[3, 40]] = 2.0
    rows.append(r); hist.append([])                         # ties across the start and the last word
    r = rng.standard_normal(n)
    r[[5, n - 2, n - 1]] = 6.0
    rows.append(r); hist.append([n - 2])                    # a tie of three, one penalised
    r = np.full(n, -np.inf)
    r[last_chunk:] = 1.0 + np.arange(n - last_chunk) * 0.125
    r[0] = 1.0
    rows.append(r); hist.append([0, w])                     # only the last thread chunk and id 0 finite
    r = rng.standard_normal(n) * 3
    r[w:] += 4.0
    rows.append(r); hist.append(list(range(w, n, 2)))       # a top-p cut through the last word
    return rows, hist


def _history(rng, n):
    """A history of random ids plus ids of the last word."""
    h = rng.integers(0, n, int(rng.integers(0, 30))).tolist()
    return h + [n - 1, _word(n)][:int(rng.integers(0, 3))]


@pytest.mark.parametrize("n_vocab", SAMPLE_VOCABS)
def test_sample_and_truncation_at_ragged_vocabularies(tmp_path, n_vocab):
    extra = _sample_extra(tmp_path, n_vocab)
    rng = np.random.default_rng(n_vocab + 3)
    base = list(_rows(rng, n_vocab))
    edges, edge_hist = _edge_rows(rng, n_vocab)
    tails, tail_hist = _tail_rows(rng, n_vocab)
    rows = np.asarray(base + edges + tails, np.float32)
    n_draws = ambiguous = in_tail = 0
    for T, rp in ((0.7, 1.1), (1.0, 1.0), (0.2, 1.5), (5.0, 1.1)):
        for top_k, top_p in _settings(n_vocab) + [(n_vocab - 1, 0.0), (n_vocab - 1, 0.95)]:
            hist = [_history(rng, n_vocab) for _ in base] + edge_hist + tail_hist
            seeds = [int(s) for s in rng.integers(0, 2 ** 63, len(rows), dtype=np.int64)]
            first_draw = int(rng.integers(0, 50))
            ids = extra.sample(rows, T, rp, seeds, first_draw, hist, top_k=top_k, top_p=top_p)
            for k in range(len(rows)):
                want, amb, keep = trunc_ref.sample(rows[k], T, rp, hist[k], sample_ref.uniform(seeds[k], first_draw),
                                                   top_k, top_p)
                n_draws += 1
                assert 0 <= ids[k] < n_vocab and keep[ids[k]], (T, rp, top_k, top_p, k, int(ids[k]))
                if amb:
                    ambiguous += 1
                    continue
                assert ids[k] == want, (T, rp, top_k, top_p, k, int(ids[k]), want)
                in_tail += int(ids[k]) >= _word(n_vocab)
    print("n_vocab %d: %d draws, %d ambiguous, %d in the last bitmap word" % (n_vocab, n_draws, ambiguous, in_tail))
    assert in_tail >= 50
    # device against device: cuts that drop nothing change no bit, and a row's id does not depend on its batch position
    for T, rp in ((0.7, 1.1), (5.0, 1.5)):
        for first_draw in (0, 7, 31):
            hist = [_history(rng, n_vocab) for _ in rows]
            seeds = [int(s) for s in rng.integers(0, 2 ** 63, len(rows), dtype=np.int64)]
            off = extra.sample(rows, T, rp, seeds, first_draw, hist)
            assert (extra.sample(rows, T, rp, seeds, first_draw, hist, top_k=n_vocab, top_p=1.0) == off).all()
            for k in range(len(rows)):
                n_fin = int(np.isfinite(rows[k]).sum())
                if n_fin < n_vocab:
                    got = extra.sample(rows[k:k + 1], T, rp, seeds[k:k + 1], first_draw, hist[k:k + 1], top_k=n_fin)
                    assert got[0] == off[k], (T, rp, k, n_fin)
            perm = rng.permutation(len(rows))
            idx = np.concatenate([perm, perm[:5]])
            for kw in (dict(top_k=40, top_p=0.95), dict(top_p=0.5), dict(top_k=n_vocab - 1)):
                a = extra.sample(rows, T, rp, seeds, first_draw, hist, **kw)
                b = extra.sample(rows[idx], T, rp, [seeds[i] for i in idx], first_draw, [hist[i] for i in idx], **kw)
                assert (b == a[idx]).all(), (T, rp, kw)
    extra.close()


# --------------------------------------------------------------------------- d. NLL
@pytest.mark.parametrize("n_vocab", SAMPLE_VOCABS)
def test_nll_at_ragged_vocabularies(tmp_path, n_vocab):
    extra = _sample_extra(tmp_path, n_vocab)
    rng = np.random.default_rng(n_vocab + 4)
    w = _word(n_vocab)
    rows = list(_rows(rng, n_vocab)) + _tail_rows(rng, n_vocab)[0]
    rows = np.asarray(rows, np.float32)
    targets = np.array([(n_vocab - 1, n_vocab // 32 * 32 if n_vocab % 32 else w, 0)[k % 3] for k in range(len(rows))],
                       np.int32)
    rows = np.concatenate([rows, rows])
    targets = np.concatenate([targets, np.roll(targets, 1)])
    got = extra.nll(rows, targets)
    want = score_ref.nll_rows(rows, targets)
    ok = score_ref.within(got, want)
    assert ok.all(), [(k, int(targets[k]), got[k], want[k]) for k in np.flatnonzero(~ok)]
    fin = np.isfinite(want)
    assert fin.sum() >= len(rows) // 2
    assert np.isfinite(want[(targets == n_vocab - 1)]).any()                 # V - 1 scored with a finite value
    err = np.abs(got[fin] - want[fin]) / np.maximum(1, np.abs(want[fin]))
    print("n_vocab %d: largest relative difference from the twin %.3g" % (n_vocab, err.max()))
    extra.close()


# --------------------------------------------------------------------------- e. the device loops at V = 32001
def _tail_model(tmp_path, kind):
    """Two slices and an extra-layers file of a 32001-id model whose output rows of the last 32 ids are scaled up (x4,
    V - 1 x8), so that the loops draw them: (slice paths, extra path, shape)."""
    paths = [str(tmp_path / "a.bin"), str(tmp_path / "b.bin")]
    base = str(tmp_path / "extra_base.bin")
    if kind == "q4_0":
        sh = ggjt.ModelShape(32001, 512, 32, 4, 3)                           # tiny128's layers
        ggjt.write_synth_slice(paths[0], sh, 0, 0, ggjt.T_Q4_0, seed=81)
        ggjt.write_synth_slice(paths[1], sh, 1, sh.n_layer - 1, ggjt.T_Q4_0, seed=81)
        ggjt.write_synth_extra(base, sh, ggjt.T_Q4_0, seed=81)
    else:
        sh = ggjt.ModelShape(32001, 512, 256, 4, 8)                          # tinyk128's layers
        ggjt.write_kquant_slice(paths[0], sh, 0, 3, "q4_K_M", seed=82)
        ggjt.write_kquant_slice(paths[1], sh, 4, sh.n_layer - 1, "q4_K_M", seed=82)
        ggjt.write_kquant_extra(base, sh, "q4_K_M", seed=82)
    extra = str(tmp_path / "extra.bin")
    v = sh.n_vocab
    _edit_output(base, str(tmp_path / "extra_x4.bin"), {r: r for r in range(v - 32, v - 1)}, 4.0)
    _edit_output(str(tmp_path / "extra_x4.bin"), extra, {v - 1: v - 1}, 8.0)
    return paths, extra, sh


@pytest.mark.parametrize("kind", ["q4_0", "q4_K_M"])
def test_device_loops_reach_the_last_ids(tmp_path, kind):
    from distributedllm_b200 import capi
    from test_gpu_score import _host_nll
    paths, extra_path, sh = _tail_model(tmp_path, kind)
    v, tail = sh.n_vocab, sh.n_vocab // 32 * 32
    n_sess, n_steps, K, P, T, rp = 4, 10, 40, 0.95, 0.9, 1.1
    gpu = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(31)
    sessions = [2, 0, 3, 1]
    prompts = [rng.integers(0, v, n).tolist() + [v - 1] for n in (4, 0, 9, 2)]
    seeds = [5, 2 ** 63 + 7, 1234, 99]

    def clear():
        for s in gpu + twin:
            s.session_clear(-1)

    # greedy
    ids = capi.generate_greedy(gpu, extra, sessions, prompts, n_steps)
    for j, k in enumerate(sessions):
        assert capi.generate_greedy(twin, extra, [k], [prompts[j]], n_steps)[:, 0].tolist() == ids[:, j].tolist(), k
        for s in twin:
            s.session_clear(k)
        assert _greedy_host(twin, extra, k, prompts[j], n_steps) == ids[:, j].tolist(), k
    assert (ids >= tail).any(), ids
    greedy = ids
    clear()
    # sampled, top_k 40 and top_p 0.95
    ids = capi.generate_sample(gpu, extra, sessions, prompts, n_steps, T, rp, seeds, top_k=K, top_p=P)
    ambiguous = 0
    for j, k in enumerate(sessions):
        alone = capi.generate_sample(twin, extra, [k], [prompts[j]], n_steps, T, rp, [seeds[j]], top_k=K, top_p=P)
        assert alone[:, 0].tolist() == ids[:, j].tolist(), k
        for s in twin:
            s.session_clear(k)
        host, safe = _sample_host_loop(twin, extra, k, prompts[j], n_steps, T, rp, seeds[j], K, P)
        assert host[:safe] == ids[:safe, j].tolist(), k
        ambiguous += safe < n_steps
    print("%s: %d sessions stopped at an ambiguous draw" % (kind, ambiguous))
    assert (ids >= tail).any(), ids
    clear()
    # score: texts that hold the last ids
    texts = [p + greedy[:, j].tolist() + [v - 1, tail - 1, v - 1] for j, p in enumerate(prompts)]
    got = capi.score(gpu, extra, sessions, texts)
    for j, k in enumerate(sessions):
        alone = capi.score(twin, extra, [k], [texts[j]])[0]
        assert (alone.view(np.uint64) == got[j].view(np.uint64)).all(), k
        for s in twin:
            s.session_clear(k)
        host = _host_nll(twin, extra, k, texts[j])
        assert np.isfinite(host).all() and score_ref.within(got[j], host).all(), k
    clear()
    # a stream: a greedy session, then a truncated sampled one joining after 3 ids
    plan = {0: (None, prompts[0], 8), 1: (seeds[1], prompts[2], 9)}
    pairs = []
    with capi.Stream(gpu, extra) as st:
        st.add(0, plan[0][1], plan[0][2])
        for pair in st:
            pairs.append(pair)
            if len(pairs) == 3:
                st.add(1, plan[1][1], plan[1][2], temperature=T, repeat_penalty=rp, seed=seeds[1], top_k=K, top_p=P)
    got = {k: [t for s, t in pairs if s == k] for k in plan}
    assert got[0] == capi.generate_greedy(twin, extra, [0], [plan[0][1]], 8)[:, 0].tolist()
    assert got[1] == capi.generate_sample(twin, extra, [1], [plan[1][1]], 9, T, rp, [seeds[1]], top_k=K, top_p=P)[:, 0].tolist()
    assert any(t >= tail for t in got[0] + got[1]), got
    extra.close()
    for s in gpu + twin:
        s.close()
