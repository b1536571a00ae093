"""The CPU oracle against the committed reference outputs (tests/golden/*.npz, produced by oracle/make_golden.py from the
UNMODIFIED reference classes).  Runs anywhere: no GPU, no reference checkout."""
import os

import numpy as np
import pytest
import torch

from mapperatorinator_b200 import tiny_dit_config, tiny_model_config
from mapperatorinator_b200.weights import init_dit_state_dict, init_model_state_dict
from oracle import cases, dit as dit_oracle, generate as gen_oracle, mel as mel_oracle, whisper as wo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def gen_gold():
    return np.load(os.path.join(GOLDEN, "generate_reference.npz"))


def test_mel_torchaudio_flavours():
    gold = np.load(os.path.join(GOLDEN, "mel_reference.npz"))
    for name, mc in cases.MEL_CASES.items():
        if mc.implementation != "torchaudio":
            continue
        out = mel_oracle.mel_forward(cases.mel_pcm(), mc).numpy()[:, ::64, :]
        scale = np.abs(gold[name]).max()
        assert np.abs(out - gold[name]).max() <= 1e-5 * scale + 1e-6


@pytest.mark.parametrize("flavour", list(cases.MODEL_FLAVOURS))
def test_encoder_and_teacher_forcing(gen_gold, flavour):
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS[flavour])
    sd = init_model_state_dict(cfg, 0)
    enc = wo.encode(sd, cfg, cases.model_pcm(cfg, 3, 0)).numpy()[:, ::32, :]
    assert np.allclose(enc, gen_gold[f"{flavour}/encoder"], rtol=1e-4, atol=2e-5)
    ids, mask = cases.teacher_forcing_case(cfg)
    logits = wo.forward_logits(sd, cfg, cases.model_pcm(cfg, 2, 1), ids, mask).numpy()[:, ::3, ::37]
    real = mask.numpy()[:, ::3]
    assert np.allclose(logits[real], gen_gold[f"{flavour}/teacher_logits"][real], rtol=1e-3, atol=2e-4)


@pytest.mark.parametrize("flavour", list(cases.MODEL_FLAVOURS))
@pytest.mark.parametrize("case", list(cases.generate_cases()))
def test_greedy_ids_bit_exact(gen_gold, layout, flavour, case):
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS[flavour])
    sd = init_model_state_dict(cfg, 0)
    prompt, neg, gk, seed = cases.generate_cases()[case]
    B = prompt.shape[0]
    mk = dict(inputs=cases.model_pcm(cfg, B, seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0), negative_prompt=neg,
              negative_prompt_attention_mask=None if neg is None else neg.ne(0))
    ids, stats = gen_oracle.model_generate(sd, cfg, layout, mk, dict(gk))
    assert np.array_equal(ids.numpy(), gen_gold[f"{flavour}/{case}/ids"])
    assert stats["generated_tokens_per_sample"] == gen_gold[f"{flavour}/{case}/counts"].tolist()


@pytest.mark.parametrize("case", list(cases.long_context_cases()))
def test_greedy_ids_long_context(gen_gold, layout, case):
    """Prompts of 150 and 600 tokens (left-padded batch of 2): the oracle against the unmodified reference's model_generate."""
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd = init_model_state_dict(cfg, 0)
    prompt, gk, seed = cases.long_context_cases()[case]
    mk = dict(inputs=cases.model_pcm(cfg, prompt.shape[0], seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
    ids, _ = gen_oracle.model_generate(sd, cfg, layout, mk, dict(gk))
    assert np.array_equal(ids.numpy(), gen_gold[f"torchaudio/{case}/ids"])


@pytest.mark.parametrize("case", list(cases.processor_cases()))
def test_processor_chain(layout, case):
    gold = np.load(os.path.join(GOLDEN, "processors_reference.npz"))
    ids_steps, gk = cases.processor_cases()[case]
    pr = gen_oracle.Processors(layout, ids_steps[0].shape[0], 3, dict(gk, types_first=True))
    for step, ids in enumerate(ids_steps):
        scores = pr(ids, cases.processor_logits(case, step, ids.shape[0], layout.vocab_size_out)).numpy()
        want = gold[f"{case}/{step}"]
        assert np.array_equal(np.isneginf(scores), np.isneginf(want)), (case, step)
        fin = np.isfinite(want)
        assert np.allclose(scores[fin], want[fin], rtol=1e-5, atol=1e-5), (case, step)


def test_dit_forward_and_loop():
    gold = np.load(os.path.join(GOLDEN, "dit_reference.npz"))
    dc = tiny_dit_config()
    sd = init_dit_state_dict(dc, 1)
    x, c, y, noise, ip, am = cases.dit_case(dc)
    out = dit_oracle.dit_forward_with_cfg(sd, dc, x, torch.tensor([37, 37]), c, y, 1.5, am).numpy()
    assert np.allclose(out, gold["forward_with_cfg"], rtol=1e-4, atol=1e-5)
    sched = dit_oracle.Schedule()
    assert sched.timestep_map == gold["timestep_map"].tolist()
    mine = np.stack([sched.sqrt_recip_alphas_cumprod, sched.sqrt_recipm1_alphas_cumprod, sched.posterior_log_variance_clipped,
                     sched.log_betas, sched.posterior_mean_coef1, sched.posterior_mean_coef2], 1)
    assert np.allclose(mine, gold["schedule"], rtol=1e-12, atol=0)
    res = dit_oracle.p_sample_loop(sd, dc, sched, x, c, y, 1.0, am, noise, inpaint_mask=ip).numpy()
    assert np.abs(res - gold["p_sample_loop"]).max() <= 2e-5


def test_dit_chunked_pipeline_loop():
    """Oracle chunk loop vs the reference's own `DiffisionPipeline.generate` (chunks with frozen / re-noised overlap, in-paint
    mask, to_positions)."""
    gold = np.load(os.path.join(GOLDEN, "dit_reference.npz"))
    dc = tiny_dit_config()
    sd = init_dit_state_dict(dc, 1)
    seq_x, seq_c, y, y_null, geo = cases.dit_chunk_case(dc)
    pos = dit_oracle.sample_sequence(sd, dc, seq_x, seq_c, y, y_null, 1.0, chunk_noise=cases.dit_chunk_noise, **geo).numpy()
    assert pos.shape == gold["chunked_positions"].shape
    assert np.abs(pos - gold["chunked_positions"]).max() <= 2e-3          # pixels (coordinates are scaled by 512 / 384)


@pytest.mark.parametrize("case", ["b1_first_window", "b1_eos_stop"])
def test_teacher_forced_check_agrees_with_generation(layout, case):
    """`teacher_forced_check` (one batched decoder pass + processor replay; what bench.py uses to check a WHOLE song against
    the oracle) must accept the oracle's own greedy output and must flag a corrupted token with its position."""
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd = init_model_state_dict(cfg, 0)
    prompt, neg, gk, seed = cases.generate_cases()[case]
    pcm = cases.model_pcm(cfg, 1, seed)
    mk = dict(inputs=pcm, decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
    ids, _ = gen_oracle.model_generate(sd, cfg, layout, mk, dict(gk))
    P = prompt.shape[1]
    rep = gen_oracle.teacher_forced_check(sd, cfg, layout, pcm, ids, P, dict(gk))
    assert rep["match"] and rep["n_checked"] == ids.shape[1] - P and rep["min_gap"] > 0
    bad = ids.clone()
    k = P + (ids.shape[1] - P) // 2
    bad[0, k] = (bad[0, k] + 1) % cfg.vocab_size_out
    rep = gen_oracle.teacher_forced_check(sd, cfg, layout, pcm, bad, P, dict(gk))
    assert not rep["match"] and rep["first_divergence"]["index"] == k and rep["first_divergence"]["gap"] > 0
