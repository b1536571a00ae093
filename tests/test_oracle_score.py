"""The CPU scoring oracle against MaiMod's scores on the unmodified reference's `server.model_forward` logits
(tests/golden/score_reference.npz, written by oracle/make_score_golden.py).  Runs anywhere: no GPU, no reference checkout."""
import os

import numpy as np
import pytest
import torch

from mapperatorinator_b200 import tiny_model_config
from mapperatorinator_b200.weights import init_model_state_dict
from oracle import cases, score
from oracle import whisper as wo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PCM_SEED = 6          # oracle/make_score_golden.py
EPS = 2e-4            # logits tolerance of the teacher-forced tests (oracle vs reference / engine)


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "score_reference.npz"))


@pytest.fixture(scope="module")
def oracle_scores():
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd = init_model_state_dict(cfg, 0)
    ids, mask = score.score_case(cfg)
    with torch.no_grad():
        logits = wo.forward_logits(sd, cfg, cases.model_pcm(cfg, ids.shape[0], PCM_SEED), ids, mask)
    return cfg, ids, mask, {k: v.numpy() for k, v in score.score_from_logits(logits, ids).items()}


def test_case_is_the_fixture_case(gold, oracle_scores):
    cfg, ids, mask, _ = oracle_scores
    assert np.array_equal(ids.numpy(), gold["ids"]) and np.array_equal(mask.numpy(), gold["mask"])
    assert mask.sum(1).tolist() == [40, 300, 700]
    assert (ids[:, 1:] >= cfg.vocab_size_out).any()             # input-only targets occur


def test_oracle_scores_equal_reference(gold, oracle_scores):
    """A logits error of EPS moves any log-softmax entry by at most 2 EPS, i.e. 2 EPS / ln 2 bits: the bound on surprisal, and
    (p-weighted) on entropy.  The argmax must agree wherever the reference's top-2 gap exceeds 2 EPS."""
    _, _, _, got = oracle_scores
    bits = 2 * EPS / np.log(2)
    for k in ("entropy", "surprisal"):
        want = gold[k]
        assert np.array_equal(np.isnan(got[k]), np.isnan(want)), k
        ok = ~np.isnan(want)
        assert np.abs(got[k][ok] - want[ok]).max() <= bits, (k, np.abs(got[k][ok] - want[ok]).max())
    assert np.array_equal(np.isnan(got["relative"]), np.isnan(gold["relative"]))
    sure = ~(gold["top2_gap"] <= 2 * EPS)                        # NaN column 0 included: -1 there on both sides
    assert np.array_equal(got["suggested"][sure], gold["suggested"][sure])


def test_fixture_edge_placements(gold):
    """Column 0 is NaN / -1; a target >= vocab_size_out has NaN surprisal and relative but a finite entropy and a suggestion."""
    V = tiny_model_config().vocab_size_out
    assert np.isnan(gold["entropy"][:, 0]).all() and (gold["suggested"][:, 0] == -1).all()
    big = np.zeros_like(gold["mask"])
    big[:, 1:] = gold["ids"][:, 1:] >= V
    assert np.isnan(gold["surprisal"][big]).all() and np.isnan(gold["relative"][big]).all()
    assert np.isfinite(gold["entropy"][:, 1:]).all() and (gold["suggested"][:, 1:] >= 0).all()
    assert np.isfinite(gold["surprisal"][:, 1:][~big[:, 1:]]).all()
