"""Beam search (`num_beams` 2..4) through the reference-facing boundary on the GPU: ids bit-exact against the unmodified reference's
`server.model_generate` (tests/golden/beam_reference.npz, which tests/test_oracle_beam.py pins the CPU oracle to), generated-token
counts equal, best-hypothesis scores within 1e-4 of the reference's `sequences_scores`."""
import os

import numpy as np
import pytest
import torch

from oracle import beam, cases

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def tiny16():
    """Tiny torchaudio model with room for 16 decoder rows (B * K, x2 under classifier-free guidance)."""
    from mapperatorinator_b200 import tiny_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd = init_model_state_dict(cfg, 0)
    return cfg, sd, B200Mapperatorinator(cfg, sd, max_windows=8, max_batch=16)


@pytest.fixture(scope="module")
def beam_gold():
    return np.load(os.path.join(GOLDEN, "beam_reference.npz"))


def _model_kwargs(cfg, prompt, neg, seed):
    return dict(inputs=cases.model_pcm(cfg, prompt.shape[0], seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0),
                negative_prompt=neg, negative_prompt_attention_mask=None if neg is None else neg.ne(0))


def _first_divergence(got: np.ndarray, want: np.ndarray):
    for b in range(min(got.shape[0], want.shape[0])):
        n = min(got.shape[1], want.shape[1])
        bad = np.flatnonzero(got[b, :n] != want[b, :n])
        if bad.size:
            t = int(bad[0])
            return f"row {b}, position {t}: got {int(got[b, t])}, want {int(want[b, t])}"
    return f"shapes {got.shape} vs {want.shape}"


@pytest.mark.parametrize("case", list(beam.beam_cases()))
def test_beam_generate_bit_exact(tiny16, layout, beam_gold, case):
    from mapperatorinator_b200.server import model_generate
    cfg, sd, model = tiny16
    prompt, neg, gk, seed = beam.beam_cases()[case]
    mk = _model_kwargs(cfg, prompt, neg, seed)
    want = beam_gold[f"{case}/ids"]
    got, stats = model_generate(model, layout, dict(mk), dict(gk))
    assert got.shape == want.shape and np.array_equal(got.numpy(), want), _first_divergence(got.numpy(), want)
    assert stats["generated_tokens_per_sample"] == beam_gold[f"{case}/counts"].tolist()
    # the best hypothesis's score, through the engine call that returns it
    B = prompt.shape[0]
    model.engine.encode(mk["inputs"].cuda(), slot_begin=0)
    ids2, scores = model.engine.generate_beams(list(range(B)), prompt, prompt.ne(0), layout, dict(gk), negative_prompt=neg,
                                               negative_mask=None if neg is None else neg.ne(0))
    assert np.array_equal(ids2.numpy(), want)
    assert np.abs(scores.numpy() - beam_gold[f"{case}/scores"]).max() <= 1e-4


def test_beam_then_greedy_same_rows_uses_greedy_graph(tiny16, layout):
    """A beam call (B = 2, K = 2: 4 decoder rows) followed by a greedy CFG call of the same row count and batch (B = 2, 4 rows) on
    one engine: the greedy call must not replay the beam call's token-step graph."""
    from mapperatorinator_b200.server import model_generate
    cfg, sd, model = tiny16
    prompt, neg, gk, seed = beam.beam_cases()["b2_leftpad_lookback_K2"]
    model_generate(model, layout, _model_kwargs(cfg, prompt, neg, seed), dict(gk))
    gold = np.load(os.path.join(GOLDEN, "generate_reference.npz"))
    prompt, neg, gk, seed = cases.generate_cases()["b2_cfg"]
    model.engine.set_option("mega", 0)
    try:
        got, _ = model_generate(model, layout, _model_kwargs(cfg, prompt, neg, seed), dict(gk))
    finally:
        model.engine.set_option("mega", 2)
    want = gold["torchaudio/b2_cfg/ids"]
    assert np.array_equal(got.numpy(), want), _first_divergence(got.numpy(), want)


def test_resident_slots_equal_per_call(tiny16, layout, beam_gold):
    """The resident path (windows encoded once into slots, then `generate(slots=...)`) gives the per-call result under beams."""
    cfg, sd, model = tiny16
    prompt, neg, gk, seed = beam.beam_cases()["b2_leftpad_lookback_K2"]
    model.engine.encode(cases.model_pcm(cfg, 2, seed).cuda(), slot_begin=5)
    got = model.engine.generate([5, 6], prompt, prompt.ne(0), layout, dict(gk))
    want = beam_gold["b2_leftpad_lookback_K2/ids"]
    assert np.array_equal(got.numpy(), want), _first_divergence(got.numpy(), want)


@pytest.mark.parametrize("bad", [dict(num_beams=5), dict(do_sample=True), dict(num_return_sequences=2), dict(length_penalty=0.5),
                                 dict(early_stopping=True)])
def test_beam_rejects_unsupported_settings(tiny16, layout, bad):
    cfg, sd, model = tiny16
    prompt, neg, gk, seed = beam.beam_cases()["b1_eos_stop_K2"]
    with pytest.raises(ValueError):
        model.engine.generate([0], prompt, prompt.ne(0), layout, dict(gk, **bad))


def test_beam_rows_must_fit_max_batch(tiny16, layout):
    cfg, sd, model = tiny16
    prompt, neg, gk, seed = beam.beam_cases()["b2_cfg_K4"]          # 2 items x 4 beams x 2 (CFG) = 16 rows fit
    prompt3 = torch.cat([prompt, prompt[:1]])
    neg3 = torch.cat([neg, neg[:1]])
    with pytest.raises(ValueError, match="max_batch"):
        model.engine.generate([0, 1, 2], prompt3, prompt3.ne(0), layout, dict(gk), negative_prompt=neg3, negative_mask=neg3.ne(0))


def _step_case(layout, K, kind, V):
    """B = 2 items x K beams of running sequences, synthetic logits of one of several shapes."""
    B, P = 2, 6
    base = [3700, 3705, 1, 9, 3645, 30, 3650, 40, 3655]
    g = torch.Generator().manual_seed(17 * K + len(kind))
    ids = torch.tensor([base] * (B * K))
    if kind != "tie":
        ids[:, -2] = torch.randint(17, 400, (B * K,), generator=g)
    L = ids.shape[1]
    gk = dict(beam.GK_BEAM, num_beams=K, max_length=L + 1 if kind == "max_length" else L + 20, lookback_time=4092.0,
              lookahead_time=3273.6, context_type="map")
    eos = layout.eos_token_ids(4092.0, 3273.6, "map")
    logits = torch.randn(B * K, V, generator=g) * 3.0
    run = torch.randn(B * K, generator=g) * 2.0
    if kind == "eos_heavy":
        logits[:, eos] += 9.0
    elif kind == "neginf_heavy":
        logits[torch.rand(B * K, V, generator=g) < 0.9] = float("-inf")
    elif kind == "tie":
        logits[:] = logits[:1]
        run[:] = 0.0
    return B, P, ids, gk, eos, logits, run


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("kind", ["plain", "eos_heavy", "neginf_heavy", "tie", "max_length"])
def test_beam_step_matches_oracle(tiny16, layout, K, kind):
    """`mb200_model_beam_step` on synthetic logits against the oracle's single step (`oracle.beam.select_step`) fed the engine's own
    processed log-probs: the first K candidates in order, the running beams (parent, token, score) and the finished store, exactly.
    The EOS set has 738 ids here, so HF keeps (1 + 738) * K candidates (2 956 at K = 4)."""
    import torch.nn.functional as F
    from oracle.generate import Processors
    cfg, sd, model = tiny16
    V = cfg.vocab_size_out
    B, P, ids, gk, eos, logits, run = _step_case(layout, K, kind, V)
    L = ids.shape[1]
    assert max(2, 1 + len(eos)) * K >= (2900 if K == 4 else 1450)
    got = model.engine.beam_step(logits.cuda(), ids, run, K, P, layout, dict(gk))
    # processed log-probs: the oracle chain on the same logits, to fp32 rounding
    want_lp = Processors(layout, B * K, P, dict(gk))(ids, F.log_softmax(logits, dim=-1))
    assert torch.equal(torch.isneginf(got["logprobs"]), torch.isneginf(want_lp))
    fin_mask = torch.isfinite(want_lp)
    assert torch.allclose(got["logprobs"][fin_mask], want_lp[fin_mask], rtol=1e-5, atol=1e-5)
    # the selection, exactly, on the engine's own log-probs
    max_length = gk["max_length"]
    running = torch.zeros(B, K, max_length, dtype=torch.long)
    running[:, :, :L] = ids.view(B, K, L)
    r = beam.select_step(got["logprobs"], running, run.view(B, K), running.clone(), torch.full((B, K), -1e9),
                         torch.zeros(B, K, dtype=torch.bool), torch.zeros(B, K, dtype=torch.long), torch.ones(B, 1, dtype=torch.bool),
                         L, P, K, torch.tensor(eos), max_length)
    assert torch.equal(got["top"].view(B, K).long(), r["order"][:, :K])
    assert torch.equal(got["parent"].view(B, K).long(), r["parent"] + torch.arange(B)[:, None] * K)
    assert torch.equal(got["token"].view(B, K), r["running"][:, :, L])
    assert torch.equal(got["score"].view(B, K), r["run_scores"])
    assert torch.equal(got["fin_flag"].view(B, K).bool(), r["fin"])
    real = r["fin"]
    assert torch.equal(got["fin_score"].view(B, K)[real], r["beam_scores"][real])
    assert torch.equal(got["fin_len"].view(B, K).long()[real], r["fin_len"][real])
    assert torch.equal(got["fin_ids"].view(B, K, L + 1)[real], r["seqs"][:, :, :L + 1][real])
    if kind == "tie":      # identical beams: the best token of every beam ties, and equal scores resolve by flat index (beam order)
        top = got["top"].view(B, K).long()
        assert torch.equal(top // V, torch.arange(K).expand(B, K)) and bool((top % V == top[:, :1] % V).all())
    if kind in ("eos_heavy", "max_length"):
        assert bool(real.any())
