"""Seeded request sets for the ragged batched generate: every case is a list of INDEPENDENT batch-1 requests (own audio window,
own prompt length, own generate_kwargs) that the engine decodes in one call.

TEST INFRASTRUCTURE.  Shared by oracle/make_ragged_golden.py (reference side, one batch-1 `model_generate` per request) and the
tests (oracle / CUDA side); fixtures only store the reference outputs.
"""
from __future__ import annotations

import torch

from .cases import GK

LB, LA = 4092.0, 3273.6


def _prompt(P: int, seed: int, sos: int = 9, tail=()) -> torch.Tensor:
    g = torch.Generator().manual_seed(1000 + seed)
    p = torch.randint(17, 3600, (1, P), generator=g)
    head = torch.tensor([3700, 3705, 1, sos])
    p[0, :min(P, 4)] = head[:P]
    if tail:
        p[0, P - len(tail):] = torch.tensor(list(tail))
    return p


def _req(prompt, gk, seed, neg=None):
    return dict(prompt=prompt, neg=neg, gk=gk, seed=seed)


def ragged_cases():
    """name -> list of requests {prompt (1, P), neg (1, Pn) | None, gk, seed (of the request's audio window)}."""
    out = {}
    # a first window (no look-back), two middle windows (`map` and `kiai`), a last window (no look-ahead)
    out["mixed_windows"] = [
        _req(_prompt(4, 1), dict(GK, max_length=4 + 20, min_new_tokens=12, lookback_time=0.0, lookahead_time=LA, context_type="map"), 21),
        _req(_prompt(9, 2), dict(GK, max_length=9 + 30, min_new_tokens=8, lookback_time=LB, lookahead_time=LA, context_type="map"), 22),
        _req(_prompt(23, 3, sos=7), dict(GK, max_length=23 + 26, min_new_tokens=16, lookback_time=LB, lookahead_time=LA, context_type="kiai"), 23),
        _req(_prompt(150, 4), dict(GK, max_length=150 + 18, min_new_tokens=18, lookback_time=LB, lookahead_time=0.0, context_type="map"), 24),
    ]
    # own stop per row: natural EOS early, max_length reached, max_length on either side of the 128-key single-split plan
    out["mixed_stops"] = [
        _req(_prompt(6, 5, tail=(3645, 30)), dict(GK, max_length=120, lookback_time=LB, lookahead_time=LA, context_type="map"), 31),
        _req(_prompt(11, 6), dict(GK, max_length=11 + 40, min_new_tokens=40, lookback_time=0.0, lookahead_time=0.0, context_type="map"), 32),
        _req(_prompt(100, 7), dict(GK, max_length=100 + 28, min_new_tokens=20, lookback_time=LB, lookahead_time=LA, context_type="map"), 33),
        _req(_prompt(110, 8), dict(GK, max_length=110 + 35, min_new_tokens=35, lookback_time=0.0, lookahead_time=LA, context_type="map"), 34),
    ]
    # the conditional temperature is decided per request (first: after a beat type -> timing temperature, second: not), look-back
    # bias on, time-shift bias on the second request only
    gt = dict(GK, lookback_time=LB, lookahead_time=0.0, context_type="timing", timing_temperature=0.1, temperature=0.9)
    out["mixed_temperature"] = [
        _req(_prompt(12, 9, sos=5, tail=(3655, 40, 3655)), dict(gt, max_length=12 + 40, min_new_tokens=40), 41),
        _req(_prompt(17, 10, sos=5, tail=(3655, 60, 3645)), dict(gt, max_length=17 + 40, min_new_tokens=40, timeshift_bias=0.7), 42),
        _req(_prompt(8, 11, sos=5, tail=(3656, 90, 3656)), dict(gt, max_length=8 + 36, min_new_tokens=36, temperature=0.7), 43),
    ]
    # classifier-free guidance on every request, own scale each (no min_new_tokens: HF masks EOS before the guidance mix, and
    # -inf - -inf there is NaN in the reference)
    p0, p1 = _prompt(7, 12, tail=(3645, 30)), _prompt(13, 13, tail=(3648, 55))
    n0, n1 = p0[:, :3].clone(), p1[:, :5].clone()
    n0[0, 0], n0[0, 2] = 0, 3712
    n1[0, 0], n1[0, 4] = 0, 3713
    out["cfg_all"] = [
        _req(p0, dict(GK, cfg_scale=1.5, max_length=7 + 24, lookback_time=0.0, lookahead_time=0.0, context_type="map"), 51, n0),
        _req(p1, dict(GK, cfg_scale=2.0, max_length=13 + 30, lookback_time=0.0, lookahead_time=LA, context_type="kiai"), 52, n1),
    ]
    return out


def model_kwargs(cfg, req) -> dict:
    """The `model_kwargs` of the batch-1 `model_generate` call of one request (prompts hold no pad id: the masks are all ones)."""
    from . import cases
    neg = req["neg"]
    return dict(inputs=cases.model_pcm(cfg, 1, req["seed"]), decoder_input_ids=req["prompt"], decoder_attention_mask=req["prompt"].ne(0),
                negative_prompt=neg, negative_prompt_attention_mask=None if neg is None else neg.ne(0))
