"""The CPU beam-search oracle against the unmodified reference's `server.model_generate(num_beams=K)` outputs
(tests/golden/beam_reference.npz, written by oracle/make_beam_golden.py).  Runs anywhere: no GPU, no reference checkout."""
import os

import numpy as np
import pytest

from mapperatorinator_b200 import tiny_model_config
from mapperatorinator_b200.weights import init_model_state_dict
from oracle import beam, cases

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def beam_gold():
    return np.load(os.path.join(GOLDEN, "beam_reference.npz"))


@pytest.fixture(scope="module")
def tiny():
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    return cfg, init_model_state_dict(cfg, 0)


@pytest.mark.parametrize("case", list(beam.beam_cases()))
def test_beam_ids_equal_reference(beam_gold, tiny, layout, case):
    cfg, sd = tiny
    prompt, neg, gk, seed = beam.beam_cases()[case]
    mk = dict(inputs=cases.model_pcm(cfg, prompt.shape[0], seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0),
              negative_prompt=neg, negative_prompt_attention_mask=None if neg is None else neg.ne(0))
    ids, stats, scores, gap = beam.beam_generate(sd, cfg, layout, mk, dict(gk))
    assert np.array_equal(ids.numpy(), beam_gold[f"{case}/ids"])
    assert stats["generated_tokens_per_sample"] == beam_gold[f"{case}/counts"].tolist()
    want = beam_gold[f"{case}/scores"]
    # the same fp32 operations in a different association order: within a few ulp of scores of magnitude ~10
    assert np.all(np.abs(scores.numpy() - want) <= 1e-6 * np.maximum(1.0, np.abs(want)))
    assert gap >= 1e-4 and abs(gap - float(beam_gold[f"{case}/min_gap"])) <= 1e-6


def test_filler_case_rows_finish_at_different_lengths(beam_gold, layout):
    """The filler rule: positions past a shorter hypothesis hold the first EOS id (pad_id 0 is falsy), which
    `generated_tokens_per_sample` counts."""
    ids = beam_gold["b2_filler_K2/ids"]
    _, _, gk, _ = beam.beam_cases()["b2_filler_K2"]
    fill = layout.eos_token_ids(gk["lookback_time"], gk["lookahead_time"], gk["context_type"])[0]
    real = [int(np.flatnonzero(r != fill).max()) + 1 for r in ids]
    assert real[0] != real[1]
    counts = beam_gold["b2_filler_K2/counts"].tolist()
    assert counts[0] == counts[1] == ids.shape[1] - 6
