"""GPU: greedy generation on the device (b200_generate_greedy), token for token against the host loop
(b200_extra_embed -> session_forward on each slice -> b200_extra_next_token), and the multi-row Q6_K lm_head against
b200_extra_logits on each row alone."""
import json
import os
import threading

import numpy as np
import pytest

from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu
REF = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_digests.json")))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _host_loop(slices, extra, session, prompt, n_steps):
    """The client's greedy loop through the host: -> (ids, hidden state of the last step)."""
    ids, toks = [], list(prompt)
    for _ in range(n_steps):
        x = extra.embed(toks)
        for s in slices:
            x = s.session_forward(session, x)
        ids.append(extra.next_token(x))
        toks = [ids[-1]]
    return ids, x


def _host_step(slices, extra, session, token):
    x = extra.embed([token])
    for s in slices:
        x = s.session_forward(session, x)
    return x


def test_config1_3b_two_slices_on_one_gpu(tmp_path):
    """BASELINE config 1 (OpenLLaMA-3B shapes, layers 0-16 / 17-25, 16-token prompt, 33 steps) as one device loop: the
    reference's greedy ids, both slices at n_past 48, and the next host step matches the host loop's bit for bit."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["3b"]
    pa, pb, extra_path = str(tmp_path / "a.bin"), str(tmp_path / "b.bin"), str(tmp_path / "extra.bin")
    ggjt.write_fast_q4_slice(pa, sh, 0, 16, seed=3)
    ggjt.write_fast_q4_slice(pb, sh, 17, 25, seed=3)
    ggjt.write_fast_q4_extra(extra_path, sh, seed=3)
    gpu = [capi.Slice(pa, 0, 512), capi.Slice(pb, 0, 512)]
    extra = capi.Extra(extra_path, 0)
    tokens = [1 + (i * 7919) % 31999 for i in range(16)]
    ids = capi.generate_greedy(gpu, extra, [0], [tokens], 33)
    assert ids.shape == (33, 1)
    assert ids[:, 0].tolist() == REF["config1"]["ids"]
    assert [s.n_past for s in gpu] == [48, 48]
    after_loop = _host_step(gpu, extra, 0, int(ids[-1, 0]))
    for s in gpu:
        s.clear_context()
    host_ids, _ = _host_loop(gpu, extra, 0, tokens, 33)
    assert host_ids == REF["config1"]["ids"]
    after_host = _host_step(gpu, extra, 0, host_ids[-1])
    assert (_bits(after_loop) == _bits(after_host)).all()
    extra.close()
    for s in gpu:
        s.close()


def _model(tmp_path, kind):
    """Two slices and an extra-layers file of one small model: (slice paths, extra path, shape)."""
    if kind == "q4_0":
        sh = ggjt.SHAPES["tiny128"]
        paths = [str(tmp_path / "a.bin"), str(tmp_path / "b.bin")]
        ggjt.write_synth_slice(paths[0], sh, 0, 0, ggjt.T_Q4_0, seed=41)
        ggjt.write_synth_slice(paths[1], sh, 1, sh.n_layer - 1, ggjt.T_Q4_0, seed=41)
        extra = str(tmp_path / "extra.bin")
        ggjt.write_synth_extra(extra, sh, ggjt.T_Q4_0, seed=41)
    elif kind == "f16":
        sh = ggjt.SHAPES["tiny"]
        paths = [str(tmp_path / "a.bin"), str(tmp_path / "b.bin")]
        ggjt.write_synth_slice(paths[0], sh, 0, 1, ggjt.T_F16, seed=42)
        ggjt.write_synth_slice(paths[1], sh, 2, sh.n_layer - 1, ggjt.T_F16, seed=42)
        extra = str(tmp_path / "extra.bin")
        ggjt.write_synth_extra(extra, sh, ggjt.T_F16, seed=42)
    else:
        sh = ggjt.SHAPES["tinyk128"]
        paths = [str(tmp_path / "a.bin"), str(tmp_path / "b.bin")]
        ggjt.write_kquant_slice(paths[0], sh, 0, 3, "q4_K_M", seed=43)
        ggjt.write_kquant_slice(paths[1], sh, 4, sh.n_layer - 1, "q4_K_M", seed=43)
        extra = str(tmp_path / "extra.bin")
        ggjt.write_kquant_extra(extra, sh, "q4_K_M", seed=43)
    return paths, extra, sh


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
def test_sessions_equal_single_session_loops_and_the_host_loop(tmp_path, kind):
    """5 sessions with different prompt lengths, two of them already mid-context, in one device loop; each session's ids
    equal a device loop of that session alone and the host loop, and the positions end where they should."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    n_sess, n_steps = 5, 10
    gpu = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(7)
    for sess, n in ((1, 7), (3, 20)):                  # mid-context sessions: the same history on both handle sets
        pre = rng.integers(0, sh.n_vocab, n).tolist()
        for hs in (gpu, twin):
            x = extra.embed(pre)
            for s in hs:
                x = s.session_forward(sess, x)
    sessions = [3, 0, 4, 1, 2]
    lengths = [5, 1, 12, 3, 9]
    prompts = [rng.integers(0, sh.n_vocab, n).tolist() for n in lengths]
    before = [s.session_n_past(k) for s in gpu for k in range(n_sess)]
    ids = capi.generate_greedy(gpu, extra, sessions, prompts, n_steps)
    assert ids.shape == (n_steps, len(sessions))
    for s in gpu:
        for j, k in enumerate(sessions):
            assert s.session_n_past(k) == before[k] + lengths[j] + n_steps - 1
    for j, k in enumerate(sessions):
        start = twin[0].session_n_past(k)
        alone = capi.generate_greedy(twin, extra, [k], [prompts[j]], n_steps)[:, 0]
        assert alone.tolist() == ids[:, j].tolist(), (kind, k)
        for s in twin:
            s.session_rewind(k, start)
        host, _ = _host_loop(twin, extra, k, prompts[j], n_steps)
        assert host == ids[:, j].tolist(), (kind, k)
        # the positions the loop left behind: one more host step on each handle set gives the same bits
        a = _host_step(gpu, extra, k, int(ids[-1, j]))
        b = _host_step(twin, extra, k, host[-1])
        assert (_bits(a) == _bits(b)).all(), (kind, k)
    assert len(set(ids.ravel().tolist())) > 3          # the run is not degenerate
    extra.close()
    for s in gpu + twin:
        s.close()


def test_multi_row_q6k_lm_head_at_7b_shape(tmp_path):
    """The Q6_K lm_head at LLaMA-7B extra-layer shape (32000 x 4096) for 1, 3, 8 and 13 rows in one call: every row's
    logits are bit-identical to b200_extra_logits on that row alone."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    path = str(tmp_path / "extra_7b.bin")
    ggjt.write_kquant_extra(path, sh, "q4_K_M", seed=44)
    extra = capi.Extra(path, 0)
    assert (extra.n_vocab, extra.n_embd) == (32000, 4096)
    rng = np.random.default_rng(8)
    for n in (1, 3, 8, 13):
        x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
        x[0] *= 0                                     # an all-zero row: Q8_K scale 0
        many = extra.logits(x)
        assert np.isfinite(many[1:]).all()
        for i in range(n):
            one = extra.logits(x[i:i + 1])
            assert (_bits(one[0]) == _bits(many[i])).all(), (n, i)
    extra.close()


def test_errors_change_nothing(tmp_models, tmp_path):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=45), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=45)]
    gpu = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    twin = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=45)
    extra = capi.Extra(extra_path, 0)
    other_path = str(tmp_path / "other.bin")           # n_embd 256
    ggjt.write_synth_slice(other_path, ggjt.SHAPES["tiny"], 0, 0, ggjt.T_Q4_0, seed=45)
    other = capi.Slice(other_path, 0, 64)
    gap = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 2, 2, seed=45), 0, 64)
    pre = list(range(3, 53))                            # session 1 at n_past 50
    for hs in (gpu, twin):
        x = extra.embed(pre)
        for s in hs:
            x = s.session_forward(1, x)

    def positions():
        return [s.session_n_past(k) for s in gpu for k in range(3)]

    before = positions()
    V = sh.n_vocab
    cases = [
        ("slices out of layer order", [gpu[1], gpu[0]], [0], [[1, 2]], 4, 1),
        ("a gap in the layers", [gpu[0], gap], [0], [[1, 2]], 4, 1),
        ("another n_embd", [other], [0], [[1, 2]], 4, 1),
        ("a handle listed twice", [gpu[0], gpu[0]], [0], [[1, 2]], 4, 1),
        ("session out of range", gpu, [3], [[1, 2]], 4, 1),
        ("session listed twice", gpu, [0, 0], [[1, 2], [3]], 4, 1),
        ("empty prompt", gpu, [0, 2], [[1, 2], []], 4, 1),
        ("negative token", gpu, [0], [[1, -1]], 4, 1),
        ("token past the vocabulary", gpu, [0], [[V]], 4, 1),
        ("no steps", gpu, [0], [[1, 2]], 0, 1),
        ("context overflow", gpu, [0, 1], [[1, 2], [5, 6, 7, 8, 9]], 11, 5),
        ("prompt overflow", gpu, [1], [[1] * 15], 1, 5),
    ]
    for what, slices, sessions, prompts, n_steps, code in cases:
        with pytest.raises(capi.B200Error) as ei:
            capi.generate_greedy(slices, extra, sessions, prompts, n_steps)
        assert ei.value.code == code, (what, str(ei.value))
        assert positions() == before, what
    # the largest loop that fits: session 1 ends exactly at n_ctx
    ids = capi.generate_greedy(gpu, extra, [0, 1], [[1, 2], [5, 6, 7, 8, 9]], 10)
    assert gpu[0].session_n_past(1) == 64 and gpu[1].session_n_past(0) == 11
    for j, (k, p) in enumerate(((0, [1, 2]), (1, [5, 6, 7, 8, 9]))):
        host, _ = _host_loop(twin, extra, k, p, 10)
        assert host == ids[:, j].tolist(), k
    a = _host_step(gpu, extra, 0, int(ids[-1, 0]))              # session 1 is full; session 0 takes one more step
    b = _host_step(twin, extra, 0, int(ids[-1, 0]))
    assert (_bits(a) == _bits(b)).all()
    extra.close()
    for s in [other, gap] + gpu + twin:
        s.close()


def test_handles_on_two_devices_or_in_a_pipeline_are_refused(tmp_models, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=46), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=46)]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=46)
    extra = capi.Extra(extra_path, 0)
    split = [capi.Slice(paths[0], 0, 64), capi.Slice(paths[1], 1, 64)]
    with pytest.raises(capi.B200Error) as ei:
        capi.generate_greedy(split, extra, [0], [[1, 2]], 3)
    assert ei.value.code == 1 and "device" in str(ei.value)
    assert [s.n_past for s in split] == [0, 0]
    # a pipeline of two ranks in this process (one thread per rank: the NCCL init waits for both)
    lib = capi.lib()
    uid = np.zeros(128, np.uint8)
    capi.check(lib.b200_pipeline_unique_id(capi._ptr(uid)))
    rcs = [None, None]

    def join(r):
        rcs[r] = lib.b200_pipeline_init(split[r].handle, r, 2, capi._ptr(uid))

    threads = [threading.Thread(target=join, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert rcs == [0, 0]
    with pytest.raises(capi.B200Error) as ei:
        capi.generate_greedy(split[:1], extra, [0], [[1, 2]], 3)
    assert ei.value.code == 1 and "pipeline" in str(ei.value)
    assert split[0].n_past == 0
    for s in split:
        capi.check(lib.b200_pipeline_destroy(s.handle))
    extra.close()
    for s in split:
        s.close()


def _serve(tmp_path):
    import distributedllm_b200.compute_node.tcp_handler as th
    from distributedllm_b200.compute_node import serve
    th._PROD = None
    srv = serve.make_server("127.0.0.1", 0, str(tmp_path / "uploads"))
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    return srv


def test_local_pipeline_generate_greedy_equals_the_node_path(tmp_path):
    """LocalPipeline.generate_greedy (device loop) against DistributedLLM.generate_greedy through a node (host loop)."""
    from distributedllm_b200.client import DistributedLLM, LocalPipeline
    from distributedllm_b200.compute_node.slices import import_llm
    from distributedllm_b200.control_center import Connection
    llm = import_llm()
    sh = ggjt.SHAPES["tiny128"]
    full = str(tmp_path / "full.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=0)
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    srv = _serve(tmp_path)
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(sl, "rb") as f:
            name = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})["file_name"]
        conn.load_slice(name)
        want = DistributedLLM([addr], extra).generate_greedy("the the a in", max_steps=12)
    finally:
        srv.shutdown()
        srv.server_close()
        llm.unload_slice()
    lp = LocalPipeline([sl], [0])
    assert lp.generate_greedy(extra, "the the a in", max_steps=12) == want
    assert lp.generate_greedy(extra, "the the a in", max_steps=12) == want      # clears the context first
    assert lp.slices[0].n_past == len(llm.tokenize_prompt(extra, "the the a in")) + 11
    lp.close()
