"""Oracle: `server.model_generate` (osuT5/osuT5/inference/server.py:83-156) and the logits-processor chain.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates, for batch rows of one `generate()` call:
  * processor order: server.py:106-134 (CFG, MonotonicTimeShift, TimeshiftBias, ConditionalTemperature | Temperature,
    LookbackBias) with HF's `MinNewTokensLengthLogitsProcessor` BEFORE them and TopK/TopP AFTER them
    (transformers 5.5.0 generation/utils.py:1129-1136,1195,1216-1224);
  * processors: osuT5/osuT5/inference/logit_processors.py:36-183;
  * CFG batch doubling with the NEGATIVE prompt in the first half: modeling_mapperatorinator.py:230-271;
  * sampling loop / EOS / pad-after-finish: transformers generation/utils.py:2743-2809;
  * token accounting: server.py:50-69.
"""
from __future__ import annotations

import time
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from . import whisper as W


class Processors:
    def __init__(self, layout, B: int, prompt_len: int, gk: dict):
        self.lay = layout
        self.B = B
        self.prompt_len = prompt_len
        self.cfg_scale = float(gk.get("cfg_scale", 1.0))
        self.timeshift_bias = float(gk.get("timeshift_bias", 0))
        self.types_first = bool(gk.get("types_first", False))
        t = float(gk.get("temperature", 1.0))
        self.temperature = t
        self.conditionals = []
        if self.types_first:   # logit_processors.py:62-71
            tt = float(gk.get("timing_temperature", t))
            mt = float(gk.get("mania_column_temperature", t))
            kt = float(gk.get("taiko_hit_temperature", t))
            if tt != t and layout.beat_type_tokens():
                self.conditionals.append((tt, set(layout.beat_type_tokens()), 1))
            if mt != t and layout.mania_type_tokens():
                self.conditionals.append((mt, set(layout.mania_type_tokens()), 3))
            if kt != t and layout.scroll_speed_tokens():
                self.conditionals.append((kt, set(layout.scroll_speed_tokens()), 1))
        self.max_offset = max([o for _, _, o in self.conditionals], default=0)
        self.lookback_time = float(gk.get("lookback_time", 0.0))
        self.lookahead_time = float(gk.get("lookahead_time", 0.0))
        self.eos_ids = layout.eos_token_ids(self.lookback_time, self.lookahead_time, gk.get("context_type"))
        self.min_new_tokens = int(gk.get("min_new_tokens") or 0)
        self.do_sample = bool(gk.get("do_sample", False))
        self.top_p = float(gk.get("top_p", 1.0) or 1.0)
        self.top_k = int(gk.get("top_k", 0) or 0)
        V = layout.vocab_size_out
        self.lookback_range = torch.zeros(V, dtype=torch.bool)
        if self.lookback_time > 0:
            self.lookback_range[layout.time_shift_start:layout.lookback_end(self.lookback_time)] = True
        self.lb_eos = torch.tensor(layout.lookback_eos_ids())
        self.timed = torch.tensor(layout.timed_token_ids())
        self.sos_ids = torch.tensor(layout.sos_ids())
        self.last_scores: Optional[torch.Tensor] = None

    def __call__(self, input_ids: torch.Tensor, logits: torch.Tensor) -> torch.Tensor:
        lay = self.lay
        s = logits.float().clone()
        # (0) HF MinNewTokensLengthLogitsProcessor (generation/logits_process.py)
        if self.min_new_tokens > 0 and input_ids.shape[1] - self.prompt_len < self.min_new_tokens:
            s[:, self.eos_ids] = float("-inf")
        # (1) CFG on raw logits: out = s[B:] + (s[:B] - s[B:]) * scale  (logits_process.py:2160-2172)
        if self.cfg_scale > 1.0:
            B = s.shape[0] // 2
            s = s[B:] + (s[:B] - s[B:]) * self.cfg_scale
        # (2) MonotonicTimeShift (logit_processors.py:136-183)
        ts0, ts1 = lay.time_shift_start, lay.time_shift_end
        L = input_ids.shape[1]
        idx = torch.arange(L)[None, :].expand_as(input_ids)
        is_ts = (input_ids >= ts0) & (input_ids < ts1)
        is_sos = torch.isin(input_ids, self.sos_ids)
        last_ts = torch.where(is_ts, idx, -1).max(dim=1).values
        last_sos = torch.where(is_sos, idx, -1).max(dim=1).values
        for b in range(input_ids.shape[0]):
            if last_ts[b] != -1 and last_ts[b] > last_sos[b]:
                val = int(input_ids[b, last_ts[b]]) - ts0
                s[b, ts0:ts0 + val] = float("-inf")
        # (3) TimeshiftBias (:36-44)
        if self.timeshift_bias != 0:
            s[:, ts0:ts1] += self.timeshift_bias
        # (4) ConditionalTemperature (:47-82) — decision from batch row 0 only; else TemperatureLogitsWarper
        temp = self.temperature
        if self.types_first and self.conditionals:
            lookback = input_ids[0, -self.max_offset:].tolist()
            for t, toks, off in self.conditionals:
                if len(lookback) >= off and lookback[-off] in toks:
                    temp = t
                    break
        s = s / temp
        # (5) LookbackBias (:85-133)
        if self.lookback_time > 0:
            scores_in = s
            if not self.types_first:
                s = s.clone()
                s[:, self.lookback_range] = float("-inf")
            else:
                if L != 0 and self.last_scores is not None:
                    last_timed = torch.isin(input_ids[:, -1], self.timed)
                    if last_timed.any():
                        last_probs = F.softmax(self.last_scores, dim=-1)
                        probs = F.softmax(s, dim=-1)
                        other = ~self.lookback_range
                        prob_eos = last_probs[:, self.lb_eos].sum(dim=-1)
                        prob_event = 1 - prob_eos
                        sc = 1 / (probs[:, other].sum(dim=-1) * prob_event + prob_eos)
                        probs[:, self.lookback_range] = 0
                        probs[:, other] *= sc.unsqueeze(1)
                        extra = torch.clip((sc - 1) * prob_eos / prob_event, 0, 1)
                        probs[:, lay.time_shift_start] = extra
                        s = torch.where(last_timed.unsqueeze(1), torch.log(probs), s)
                self.last_scores = scores_in
        # (6) HF warpers, sampling only
        if self.do_sample:
            if self.top_k:
                k = min(self.top_k, s.shape[-1])
                s = s.masked_fill(s < torch.topk(s, k)[0][..., -1, None], float("-inf"))
            if self.top_p < 1.0:
                sl, si = torch.sort(s, descending=False)
                cum = sl.softmax(dim=-1).cumsum(dim=-1)
                rm = cum <= (1 - self.top_p)
                rm[..., -1:] = False
                s = s.masked_fill(rm.scatter(1, si, rm), float("-inf"))
        return s


def model_generate(w, cfg, layout, model_kwargs: dict, generate_kwargs: dict, position_rule: str = "arange",
                   return_trace: bool = False, enc: Optional[torch.Tensor] = None):
    """Same signature/returns as the reference `model_generate` with (model, tokenizer) replaced by (w, cfg, layout)."""
    gk = dict(generate_kwargs)
    pcm = model_kwargs["inputs"]
    ids = model_kwargs["decoder_input_ids"].long()
    B, P = ids.shape
    mask = model_kwargs.get("decoder_attention_mask")
    mask = torch.ones_like(ids, dtype=torch.bool) if mask is None else mask.bool()
    neg = model_kwargs.get("negative_prompt")
    neg_mask = model_kwargs.get("negative_prompt_attention_mask")
    pr = Processors(layout, B, P, gk)
    max_length = int(gk.get("max_length", cfg.tgt_seq_len))
    pad_id = gk.get("pad_token_id", layout.pad_id)
    eos = torch.tensor(pr.eos_ids)
    use_cfg = neg is not None and pr.cfg_scale > 1.0
    t0 = time.perf_counter()
    if enc is None:
        enc = W.encode(w, cfg, pcm)
    if use_cfg:   # prepare_inputs_for_generation: first half carries the negative prompt
        enc2 = enc.repeat(2, 1, 1)
        ids2 = ids.repeat(2, 1); ids2[:B, :neg.shape[1]] = neg
        # NB `negative_prompt_attention_mask` never reaches prepare_inputs_for_generation: HF `generate()` has a parameter of
        # that exact name (transformers generation/utils.py:2142) and swallows it, so the negative-prompt rows run with the
        # CONDITIONAL prompt's padding mask (pinned by tests/golden b2_cfg).  Mirrored, not "fixed".
        mask2 = mask.repeat(2, 1)
        st = W.DecoderState(w, cfg, enc2)
        logits = W.decoder_forward(st, ids2, mask2, position_rule, last_only=True)[:, -1]
    else:
        st = W.DecoderState(w, cfg, enc)
        logits = W.decoder_forward(st, ids, mask, position_rule, last_only=True)[:, -1]
    unfinished = torch.ones(B, dtype=torch.long)
    trace = []
    gen = torch.Generator().manual_seed(int(gk.get("seed", 0)))
    while True:
        scores = pr(ids, logits)
        if return_trace:
            trace.append((logits.clone(), scores.clone()))
        if pr.do_sample:
            nxt = torch.multinomial(F.softmax(scores, dim=-1), 1, generator=gen).squeeze(1)
        else:
            nxt = torch.argmax(scores, dim=-1)
        nxt = nxt * unfinished + pad_id * (1 - unfinished)
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        unfinished = unfinished & ~torch.isin(nxt, eos).long()
        if ids.shape[1] >= max_length:
            unfinished = unfinished * 0
        if unfinished.max() == 0:
            break
        step_ids = nxt[:, None]
        if use_cfg:
            step_ids = step_ids.repeat(2, 1)
        logits = W.decoder_forward(st, step_ids, None, position_rule)[:, -1]
    elapsed = time.perf_counter() - t0
    prompt_counts = mask.long().sum(-1)
    out_counts = ids.ne(pad_id).long().sum(-1)
    gen_counts = torch.clamp(out_counts - prompt_counts, min=0)
    n = int(gen_counts.sum())
    stats = {"generated_tokens": n, "generated_tokens_per_sample": gen_counts.tolist(),
             "elapsed_seconds": float(elapsed), "tokens_per_second": n / elapsed if elapsed > 0 else 0.0}
    if return_trace:
        return ids, stats, trace
    return ids, stats


def teacher_forced_check(w, cfg, layout, pcm: torch.Tensor, full_ids: torch.Tensor, prompt_len: int, generate_kwargs: dict,
                         position_rule: str = "arange", enc: Optional[torch.Tensor] = None) -> dict:
    """Greedy-parity check of a FINISHED generation without re-running the token loop: ONE teacher-forced decoder pass over
    `full_ids` (B = 1, prompt + generated), then the processor chain replayed position by position on those logits
    (server.py:106-134 order, same `Processors` as `model_generate`).  For every generated position t it asks whether
    argmax(processed scores) == full_ids[t] and records the smallest top-1 / top-2 gap seen, so a disagreement can be told apart
    from a near-tie.  Returns {"match", "n_checked", "first_divergence": None | {"index", "got", "want", "gap"}, "min_gap",
    "gaps", "mismatch"}: the top-1 / top-2 gap of every generated position and whether its token differs from the argmax.
    Greedy only (do_sample False), cfg_scale 1."""
    gk = dict(generate_kwargs)
    assert not gk.get("do_sample", False) and float(gk.get("cfg_scale", 1.0)) <= 1.0
    ids = full_ids.long()
    assert ids.dim() == 2 and ids.shape[0] == 1
    L = ids.shape[1]
    if enc is None:
        enc = W.encode(w, cfg, pcm)
    st = W.DecoderState(w, cfg, enc)
    mask = torch.ones(1, L - 1, dtype=torch.bool)
    mask[:, :prompt_len] = ids[:, :prompt_len].ne(layout.pad_id)
    logits = W.decoder_forward(st, ids[:, :L - 1], mask, position_rule)             # (1, L-1, V): row t-1 predicts token t
    pr = Processors(layout, 1, prompt_len, gk)
    first, min_gap, gaps, mismatch = None, float("inf"), [], []
    for t in range(prompt_len, L):
        scores = pr(ids[:, :t], logits[:, t - 1])
        top = torch.topk(scores[0], 2)
        gap = float(top.values[0] - top.values[1])
        min_gap = min(min_gap, gap)
        gaps.append(gap)
        want = int(top.indices[0])
        mismatch.append(want != int(ids[0, t]))
        if want != int(ids[0, t]) and first is None:
            got_score = float(scores[0, int(ids[0, t])])
            first = {"index": t, "got": int(ids[0, t]), "want": want, "gap": float(top.values[0]) - got_score}
    return {"match": first is None, "n_checked": L - prompt_len, "first_divergence": first, "min_gap": min_gap, "gaps": gaps,
            "mismatch": mismatch}
