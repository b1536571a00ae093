"""Stage-level parity through the reference-facing boundary: CUDA engine vs the CPU oracle AND vs the committed reference
outputs (tests/golden, produced from the unmodified reference classes), on the same seeded inputs.
Tolerances: greedy token ids bit-exact; fp32 tensors 1e-4 (encoder) / 2e-4 (logits); diffusion coordinates 1e-3 abs (north_star)."""
import os

import numpy as np
import pytest
import torch

from oracle import cases

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", params=["nnAudio", "torchaudio"])
def tiny(request):
    from mapperatorinator_b200 import tiny_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS[request.param])
    sd = init_model_state_dict(cfg, 0)
    return request.param, cfg, sd, B200Mapperatorinator(cfg, sd, max_windows=8, max_batch=8)


@pytest.fixture(scope="module")
def gen_gold():
    return np.load(os.path.join(GOLDEN, "generate_reference.npz"))


def test_encoder_states(tiny, gen_gold):
    from oracle import whisper as wo
    flavour, cfg, sd, model = tiny
    pcm = cases.model_pcm(cfg, 3, 0)
    ref = wo.encode(sd, cfg, pcm)
    out = model.engine.encode(pcm.cuda(), 0, return_states=True).cpu()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-4), (out - ref).abs().max()
    assert np.allclose(out.numpy()[:, ::32, :], gen_gold[f"{flavour}/encoder"], rtol=1e-4, atol=1e-4)


def test_teacher_forced_logits_left_padded(tiny, gen_gold):
    from mapperatorinator_b200.server import model_forward
    from oracle import whisper as wo
    flavour, cfg, sd, model = tiny
    pcm = cases.model_pcm(cfg, 2, 1)
    ids, mask = cases.teacher_forcing_case(cfg)
    ref = wo.forward_logits(sd, cfg, pcm, ids, mask)
    out = model_forward(model, dict(inputs=pcm, decoder_input_ids=ids, decoder_attention_mask=mask), dict(precision="fp32"))
    real = mask[:, :, None].expand_as(ref)
    assert torch.allclose(out[real], ref[real], rtol=2e-4, atol=2e-4), (out[real] - ref[real]).abs().max()
    g = gen_gold[f"{flavour}/teacher_logits"]
    r3 = mask.numpy()[:, ::3]
    assert np.allclose(out.numpy()[:, ::3, ::37][r3], g[r3], rtol=1e-3, atol=3e-4)


MEGA_MODE = {"megakernel": 1, "dataflow": 2, "graph": 0, "graph_pdl": 0}


@pytest.mark.parametrize("path", ["dataflow", "megakernel", "graph", "graph_pdl"])
@pytest.mark.parametrize("case", list(cases.generate_cases()))
def test_greedy_generate_bit_exact(tiny, layout, gen_gold, case, path):
    """Every token-loop driver (dataflow megakernel = tagged-pair exchange, no grid barrier; grid-barrier megakernel; CUDA-graph
    replay, with and without programmatic dependent launch) must reproduce the reference's greedy ids exactly: prompts with left
    padding, look-back bias, natural EOS stop, time-shift bias + batch-row-0 conditional temperature, classifier-free guidance."""
    from mapperatorinator_b200.server import model_generate
    from oracle import generate as go
    flavour, cfg, sd, model = tiny
    model.engine.set_option("mega", MEGA_MODE[path])
    model.engine.set_option("pdl", 1 if path == "graph_pdl" else 0)
    prompt, neg, gk, seed = cases.generate_cases()[case]
    B = prompt.shape[0]
    mk = dict(inputs=cases.model_pcm(cfg, B, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0), negative_prompt=neg,
              negative_prompt_attention_mask=None if neg is None else neg.ne(0))
    want, wstats = go.model_generate(sd, cfg, layout, dict(mk), dict(gk))
    try:
        got, gstats = model_generate(model, layout, dict(mk), dict(gk))
    finally:
        model.engine.set_option("mega", 2)
        model.engine.set_option("pdl", 0)
    assert got.shape == want.shape, (got.shape, want.shape)
    if not torch.equal(got, want):
        r, c = (got != want).nonzero()[0].tolist()
        pytest.fail(f"first divergence vs oracle at row {r} col {c}: got {got[r, c].item()} want {want[r, c].item()}")
    assert gstats["generated_tokens_per_sample"] == wstats["generated_tokens_per_sample"]
    assert np.array_equal(got.numpy(), gen_gold[f"{flavour}/{case}/ids"]), "differs from the reference fixture"


@pytest.mark.parametrize("path", ["dataflow", "megakernel", "graph"])
@pytest.mark.parametrize("case", list(cases.long_context_cases()))
def test_greedy_generate_long_context(tiny, layout, gen_gold, case, path):
    """Contexts beyond 128 tokens switch the self-attention cache to 64-key splits merged by the last-arriving split (3 splits at
    174 tokens; 10 splits at 612 tokens = the rolled many-split merge).  Checked against the oracle AND the reference fixture
    (tests/golden, unmodified `server.model_generate`)."""
    from mapperatorinator_b200.server import model_generate
    from oracle import generate as go
    flavour, cfg, sd, model = tiny
    prompt, gk, seed = cases.long_context_cases()[case]
    mk = dict(inputs=cases.model_pcm(cfg, 2, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
    want, _ = go.model_generate(sd, cfg, layout, dict(mk), dict(gk))
    model.engine.set_option("mega", MEGA_MODE[path])
    try:
        got, _ = model_generate(model, layout, dict(mk), dict(gk))
    finally:
        model.engine.set_option("mega", 2)
    assert got.shape == want.shape
    if not torch.equal(got, want):
        r, c = (got != want).nonzero()[0].tolist()
        pytest.fail(f"first divergence vs oracle at row {r} col {c}: got {got[r, c].item()} want {want[r, c].item()}")
    assert np.array_equal(got.numpy(), gen_gold[f"{flavour}/{case}/ids"]), "differs from the reference fixture"


def test_sampling_is_valid_and_seeded(tiny, layout):
    from mapperatorinator_b200.server import model_generate
    _, cfg, sd, model = tiny
    prompt = torch.tensor([[3700, 3705, 1, 9]])
    gk = dict(cases.GK, do_sample=True, top_p=0.9, max_length=4 + 32, min_new_tokens=32, lookback_time=0.0, lookahead_time=0.0,
              context_type="map", seed=5)
    mk = dict(inputs=cases.model_pcm(cfg, 1), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
    a, _ = model_generate(model, layout, dict(mk), dict(gk))
    b, _ = model_generate(model, layout, dict(mk), dict(gk))
    c, _ = model_generate(model, layout, dict(mk), dict(gk, seed=6))
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert int(a[:, 4:].max()) < cfg.vocab_size_out and a.shape == (1, 36)


def _chain_case(layout, cfg, B, seed):
    """Two consecutive selection steps on synthetic logits: ids0 (prompt with a time shift after SOS -> MonotonicTimeShift active),
    then ids1 = ids0 + one token per row (row 0: a TIMED type token -> the LookbackBias branch fires; row 1: a plain time shift)."""
    g = torch.Generator().manual_seed(seed)
    V = cfg.vocab_size_out
    ts0 = layout.time_shift_start
    timed = sorted(layout.timed_token_ids())[3]
    rows = [[3700, 3705, 1, 9, timed, ts0 + 40, 3601], [3701, 3706, 1, 9, timed, ts0 + 12, 3602], [3702, 3707, 1, 9, timed, ts0 + 300, 3603]][:B]
    ids0 = torch.tensor(rows)
    nxt = torch.tensor([[timed], [ts0 + 44], [timed]][:B])
    ids1 = torch.cat([ids0, nxt], 1)
    return ids0, ids1, torch.randn(B, V, generator=g) * 2.5, torch.randn(B, V, generator=g) * 2.5


@pytest.mark.parametrize("top_k,top_p", [(0, 0.95), (50, 0.95), (50, 1.0), (0, 0.9), (0, 1.0)])
@pytest.mark.parametrize("B", [1, 3])
def test_sampling_chain_keep_set_matches_oracle(tiny, layout, top_k, top_p, B):
    """The reference's production mode (configs/inference/default.yaml:45-56: do_sample, top_p 0.95) through the fused chain vs
    `oracle.generate.Processors` (pinned branch by branch to the reference processors + HF warpers): the set of ids that survive
    MinNewTokens / MonotonicTimeShift / LookbackBias / TopK / TopP must be IDENTICAL, the renormalised probabilities equal to 1e-6,
    and the drawn token must lie in the keep-set.  Two consecutive steps, so LookbackBias runs with real `last_scores`."""
    from oracle import generate as go
    _, cfg, sd, model = tiny
    ids0, ids1, l0, l1 = _chain_case(layout, cfg, B, 100 * top_k + B)
    P = 4
    gk = dict(cases.GK, do_sample=True, top_p=top_p, top_k=top_k, max_length=64, min_new_tokens=8, lookback_time=4092.0, lookahead_time=3273.6,
              context_type="map", seed=1234)
    pr = go.Processors(layout, B, P, gk)
    for step, (ids, lg) in enumerate(((ids0, l0), (ids1, l1))):
        want = pr(ids, lg)
        got, chosen = model.engine.logits_chain(lg.cuda(), ids, P, layout, gk, step=step, has_last_scores=step > 0)
        got = got.cpu()
        keep_w, keep_g = want != float("-inf"), got != float("-inf")
        pw, pg = torch.softmax(want, -1), torch.softmax(got, -1)
        # Exact keep-set, except ids whose probability is below 1e-9 on BOTH sides: LookbackBias writes log(clip((s - 1) P_eos / P_ev, 0, 1))
        # at the first time-shift id, and with a peaked distribution s - 1 is a one-ulp quantity (6e-8 or exactly 0), so that id sits at
        # probability 5e-12 or -inf depending on the last rounding; it can never be drawn either way.
        relevant = (pw > 1e-9) | (pg > 1e-9)
        bad = (keep_w != keep_g) & relevant
        assert not bad.any(), f"step {step}: keep-sets differ at {bad.nonzero()[:5].tolist()} (|want|={int(keep_w.sum())}, |got|={int(keep_g.sum())})"
        assert int((keep_w != keep_g).sum()) <= B, "more than one knife-edge id per row"
        assert (pw - pg).abs().max() <= 1e-6, (pw - pg).abs().max()
        for b in range(B):
            assert keep_w[b, int(chosen[b])], f"step {step} row {b}: drew id {int(chosen[b])} outside the keep-set"
    if top_p < 1.0:
        assert int(keep_w.sum()) < B * cfg.vocab_size_out            # the warpers did remove something


def test_sampler_follows_the_processed_distribution(tiny, layout):
    """Chi-square test of the device sampler (inverse CDF over the kept entries, splitmix64 counter RNG): 3 000 independent seeds on one
    fixed distribution (top_k = 6) against the oracle's probabilities.  5 degrees of freedom: chi2 < 25.7 at p = 1e-4."""
    from oracle import generate as go
    _, cfg, sd, model = tiny
    ids0, _, l0, _ = _chain_case(layout, cfg, 1, 9)
    gk = dict(cases.GK, do_sample=True, top_p=1.0, top_k=6, max_length=64, lookback_time=0.0, lookahead_time=0.0, context_type="map")
    want = go.Processors(layout, 1, 4, gk)(ids0, l0)
    probs = torch.softmax(want, -1)[0]
    support = (probs > 0).nonzero().flatten().tolist()
    assert len(support) == 6
    counts = {i: 0 for i in support}
    n = 3000
    lg = l0.cuda()
    for seed in range(n):
        _, chosen = model.engine.logits_chain(lg, ids0, 4, layout, dict(gk, seed=seed), step=0)
        counts[int(chosen[0])] += 1                                   # KeyError = a draw outside the support
    chi2 = sum((counts[i] - n * float(probs[i])) ** 2 / (n * float(probs[i])) for i in support)
    assert chi2 < 25.7, (chi2, counts, [float(probs[i]) for i in support])


def test_sampling_uses_a_fresh_seed_per_call(tiny, layout):
    """Without an explicit `seed` the engine draws one per call from torch's default generator (the reference samples from torch's
    global RNG): two calls differ, `torch.manual_seed` reproduces them."""
    from mapperatorinator_b200.server import model_generate
    _, cfg, sd, model = tiny
    prompt = torch.tensor([[3700, 3705, 1, 9]])
    gk = dict(cases.GK, do_sample=True, top_p=0.95, max_length=4 + 32, min_new_tokens=32, lookback_time=0.0, lookahead_time=0.0, context_type="map")
    mk = dict(inputs=cases.model_pcm(cfg, 1), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
    torch.manual_seed(99)
    a, _ = model_generate(model, layout, dict(mk), dict(gk))
    b, _ = model_generate(model, layout, dict(mk), dict(gk))
    torch.manual_seed(99)
    a2, _ = model_generate(model, layout, dict(mk), dict(gk))
    assert not torch.equal(a, b) and torch.equal(a, a2)


def test_song_decoder_equals_per_window_calls(tiny, layout):
    """Resident-encoder sequential loop (pipeline.SongDecoder, SURVEY N1) == the reference call pattern (one model_generate
    per window, encoder re-run each time)."""
    from mapperatorinator_b200.pipeline import SongDecoder
    from mapperatorinator_b200.server import model_generate
    _, cfg, sd, model = tiny
    n = 4
    windows = cases.model_pcm(cfg, n, 9)
    base = [3700, 3705, 1, 9]
    prompt_fn = lambda i, streams: base if i == 0 else base + streams[i - 1][-8:]
    gk_fn = lambda i: dict(cases.GK, max_length=(4 if i == 0 else 12) + 16, min_new_tokens=16, lookback_time=4092.0 if i else 0.0,
                           lookahead_time=3273.6 if i < n - 1 else 0.0, context_type="map")
    song = SongDecoder(model, layout)
    song.encode_song(windows.cuda())
    a = song.decode_windows(n, prompt_fn, gk_fn)
    b = []
    for i in range(n):
        p = torch.tensor([prompt_fn(i, b)])
        ids, _ = model_generate(model, layout, dict(inputs=windows[i:i + 1], decoder_input_ids=p, decoder_attention_mask=p.ne(0)), gk_fn(i))
        b.append(ids[0, p.shape[1]:].tolist())
    assert a == b and all(len(s) == 16 for s in a)


# ---- DiT --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_dit():
    from mapperatorinator_b200 import tiny_dit_config
    from mapperatorinator_b200.diffusion import B200DiT
    from mapperatorinator_b200.weights import init_dit_state_dict
    dc = tiny_dit_config()
    sd = init_dit_state_dict(dc, 1)
    return dc, sd, B200DiT(dc, sd, max_seq_len=512)


@pytest.mark.parametrize("T,mask", [(300, "band"), (100, "none"), (130, "dense")])
def test_dit_forward_with_cfg(tiny_dit, T, mask):
    from oracle import dit as do
    dc, sd, dit = tiny_dit
    x, c, y, _, _, _ = cases.dit_case(dc, T, seed=2)
    g = torch.Generator().manual_seed(T)
    am = {"band": do.band_mask(T, 128), "none": None, "dense": torch.rand(T, T, generator=g) < 0.2}[mask]
    if mask == "dense":
        am[torch.arange(T), torch.arange(T)] = False
    t = torch.tensor([37, 37])
    ref = do.dit_forward_with_cfg(sd, dc, x, t, c, y, 1.5, am)
    out = dit.forward_with_cfg(x.cuda(), t, c.cuda(), y.cuda(), 1.5, attn_mask=None if am is None else am.cuda()).cpu()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-4), (out - ref).abs().max()


def test_dit_sample_loop_both_seams(tiny_dit):
    from mapperatorinator_b200.diffusion import InpaintDenoiser, create_diffusion
    from oracle import dit as do
    gold = np.load(os.path.join(GOLDEN, "dit_reference.npz"))
    dc, sd, dit = tiny_dit
    x, c, y, noise, ip, am = cases.dit_case(dc)
    fw = dit.forward_with_cfg(x.cuda(), torch.tensor([37, 37]), c.cuda(), y.cuda(), 1.5, attn_mask=am.cuda()).cpu().numpy()
    assert np.allclose(fw, gold["forward_with_cfg"], rtol=1e-4, atol=1e-4)
    diff = create_diffusion([100, 0, 0, 0, 0, 0, 0, 0, 0, 0], "squaredcos_cap_v2", 1000)
    ref = do.p_sample_loop(sd, dc, do.Schedule(), x, c, y, 1.0, am, noise, inpaint_mask=ip)
    mk = dict(c=c.cuda(), y=y.cuda(), cfg_scale=1.0, attn_mask=am.cuda(), key_padding_mask=None)
    fused = diff.p_sample_loop(dit.forward_with_cfg, x.shape, x.cuda(), denoised_fn=InpaintDenoiser(ip.cuda(), x.cuda()),
                               clip_denoised=True, model_kwargs=mk, step_noise=noise.cuda()).cpu()
    assert (fused - ref).abs().max() <= 1e-3, (fused - ref).abs().max()              # north_star tolerance: 1e-3 abs
    assert np.abs(fused.numpy() - gold["p_sample_loop"]).max() <= 1e-3                # ... and against the reference's own loop
    zc, ipc = x.cuda(), ip.cuda()
    closure = lambda xx: torch.where(ipc, xx, zc)                                      # arbitrary host callable -> Python-loop seam
    loop = diff.p_sample_loop(dit.forward_with_cfg, x.shape, x.cuda(), denoised_fn=closure, clip_denoised=True, model_kwargs=mk,
                              step_noise=noise.cuda()).cpu()
    assert (loop - ref).abs().max() <= 1e-3


def test_dit_chunked_sample_sequence(tiny_dit):
    """`diffusion.sample_sequence` (the slider-free body of DiffisionPipeline.generate, fused loop per chunk) vs the reference
    pipeline's own output: 1e-3 in normalised coordinates = 0.256 px in x."""
    from mapperatorinator_b200.diffusion import sample_sequence
    gold = np.load(os.path.join(GOLDEN, "dit_reference.npz"))
    dc, sd, dit = tiny_dit
    seq_x, seq_c, y, y_null, geo = cases.dit_chunk_case(dc)
    shapes = []
    T, ob, ms = seq_x.shape[1], geo["overlap_buffer"], geo["max_seq_len"]
    for i in range(0, T - ob * 2, ms - ob * 2):
        shapes.append((2, 2, min(i + ms, T) - i))
    noise = [cases.dit_chunk_noise(k, s).cuda() for k, s in enumerate(shapes)]
    pos = sample_sequence(dit, seq_x, seq_c, y, y_null, 1.0, step_noise=noise, **geo).cpu().numpy()
    assert np.abs(pos - gold["chunked_positions"]).max() <= 0.256
