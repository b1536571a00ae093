"""Oracle: `server.model_generate` with `num_beams > 1` (HF `generate(num_beams=K, do_sample=False)` -> `_beam_search`).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates, with explicit per-row decoder caches:
  * transformers 5.5.0 generation/utils.py:3076-3380 (the loop) and :2856-3075 (top-k continuations, running beams,
    finished-hypothesis update with length penalty and -1e9 sentinels, early-stop heuristic with early_stopping=False);
  * the processor chain of oracle/generate.py applied to LOG-PROBS (log_softmax first, as `_beam_search` does);
  * `MapperatorinatorCache.reorder_cache` (osuT5/osuT5/inference/cache_utils.py:16-20): under CFG the self-attention cache is
    reordered with `beam_idx.repeat(2)`, so the conditional rows take the NEGATIVE rows' history.  Mirrored, not "fixed";
  * `LookbackBiasLogitsWarper.last_scores` is indexed by row position and is not reordered (the same `Processors` object is
    called with the rows in position order every step);
  * the output filler: `pad_token_id or eos_token_id[0]`, i.e. the first EOS id when pad_id is 0.
Candidate order on equal scores: score descending, then flat index (beam * V + token) ascending.
"""
from __future__ import annotations

import time
from typing import Optional

import torch
import torch.nn.functional as F

from . import whisper as W
from .generate import Processors

GK_BEAM = dict(precision="fp32", do_sample=False, top_p=0.9, top_k=0, cfg_scale=1.0, timeshift_bias=0, types_first=True,
               temperature=0.9, timing_temperature=0.1, mania_column_temperature=0.5, taiko_hit_temperature=0.5)


def _sort_desc(x: torch.Tensor) -> torch.Tensor:
    return torch.sort(x, dim=-1, descending=True, stable=True).indices


def _adjacent_gap(v: torch.Tensor) -> float:
    """smallest difference between neighbours of a descending, finite-filtered row set"""
    g = float("inf")
    for row in v:
        row = row[torch.isfinite(row)]
        if row.numel() > 1:
            g = min(g, float((row[:-1] - row[1:]).min()))
    return g


def select_step(lp, running, run_scores, seqs, beam_scores, fin, fin_len, unsat, cur_len: int, P: int, K: int, eos: torch.Tensor,
                max_length: int) -> dict:
    """One step of `_beam_search` after the processor chain: lp (B*K, V) processed log-probs, running (B, K, max_length) sequences,
    run_scores (B, K); the finished store seqs / beam_scores / fin / fin_len (B, K[, max_length]); unsat (B, 1) the early-stop
    heuristic's state.  Returns the kept candidates (order, topv, hits), the new running beams (running, run_scores, parent = beam
    within the item) and the new finished store."""
    B = running.shape[0]
    V = lp.shape[-1]
    btk = max(2, 1 + eos.numel()) * K
    top_mask = torch.arange(btk) < K
    acc = (lp.view(B, K, V) + run_scores[:, :, None]).reshape(B, K * V)
    order = _sort_desc(acc)[:, :btk]
    topv = torch.gather(acc, 1, order)
    cand_beam, cand_tok = order // V, order % V
    topk_seqs = torch.gather(running, 1, cand_beam[:, :, None].expand(B, btk, max_length)).clone()
    topk_seqs[:, :, cur_len] = cand_tok
    hits = torch.isin(cand_tok, eos) | (cur_len + 1 >= max_length)
    run_vals = topv + hits.to(torch.float32) * -1.0e9
    nxt = _sort_desc(run_vals)[:, :K]
    running = torch.gather(topk_seqs, 1, nxt[:, :, None].expand(B, K, max_length))
    run_scores = torch.gather(run_vals, 1, nxt)
    parent = torch.gather(cand_beam, 1, nxt)
    # finished hypotheses (length_penalty 1.0: python int ** 1.0 -> a float scalar; early_stopping False)
    did = hits & top_mask[None, :]
    s = topv / float((cur_len + 1 - P) ** 1.0)
    s = s + (~unsat).to(torch.float32) * -1.0e9
    s = s + (~did) * -1.0e9
    m_scores = torch.cat([beam_scores, s], 1)
    m_seqs = torch.cat([seqs, topk_seqs], 1)
    m_fin = torch.cat([fin, did], 1)
    m_len = torch.cat([fin_len, torch.full((B, btk), cur_len + 1 - P, dtype=torch.long)], 1)
    sel = _sort_desc(m_scores)[:, :K]
    beam_scores = torch.gather(m_scores, 1, sel)
    seqs = torch.gather(m_seqs, 1, sel[:, :, None].expand(B, K, max_length))
    fin = torch.gather(m_fin, 1, sel)
    fin_len = torch.gather(m_len, 1, sel)
    return dict(order=order, topv=topv, hits=hits, running=running, run_scores=run_scores, parent=parent, seqs=seqs,
                beam_scores=beam_scores, fin=fin, fin_len=fin_len)


def beam_generate(w, cfg, layout, model_kwargs: dict, generate_kwargs: dict, position_rule: str = "arange",
                  enc: Optional[torch.Tensor] = None):
    """Returns (ids (B, L), stats, scores (B,) = the best hypothesis's length-normalised score, min_gap).
    `min_gap` is the smallest score difference, over all steps, between neighbours in the orders that decide the outcome:
    the first K+1 candidates (finished hypotheses), the first K+1 non-stopping candidates (running beams)."""
    gk = dict(generate_kwargs)
    K = int(gk.get("num_beams", 1))
    pcm = model_kwargs["inputs"]
    ids = model_kwargs["decoder_input_ids"].long()
    B, P = ids.shape
    mask = model_kwargs.get("decoder_attention_mask")
    mask = torch.ones_like(ids, dtype=torch.bool) if mask is None else mask.bool()
    neg = model_kwargs.get("negative_prompt")
    pr = Processors(layout, B * K, P, gk)
    max_length = int(gk.get("max_length", cfg.tgt_seq_len))
    pad_id = gk.get("pad_token_id", layout.pad_id)
    fill = pad_id or pr.eos_ids[0]
    eos = torch.tensor(pr.eos_ids)
    use_cfg = neg is not None and pr.cfg_scale > 1.0
    BK = B * K
    t0 = time.perf_counter()
    if enc is None:
        enc = W.encode(w, cfg, pcm)
    # _expand_inputs_for_generation: every per-item tensor repeat_interleave(K)
    enc_k, ids_k, mask_k = enc.repeat_interleave(K, 0), ids.repeat_interleave(K, 0), mask.repeat_interleave(K, 0)
    if use_cfg:
        neg_k = neg.long().repeat_interleave(K, 0)
        ids2 = ids_k.repeat(2, 1); ids2[:BK, :neg_k.shape[1]] = neg_k
        st = W.DecoderState(w, cfg, enc_k.repeat(2, 1, 1))
        logits = W.decoder_forward(st, ids2, mask_k.repeat(2, 1), position_rule, last_only=True)[:, -1]
    else:
        st = W.DecoderState(w, cfg, enc_k)
        logits = W.decoder_forward(st, ids_k, mask_k, position_rule, last_only=True)[:, -1]
    V = logits.shape[-1]

    running = torch.full((B, K, max_length), fill, dtype=torch.long)
    running[:, :, :P] = ids_k.view(B, K, P)
    seqs = running.clone()
    run_scores = torch.zeros(B, K); run_scores[:, 1:] = -1e9
    beam_scores = torch.full((B, K), -1e9)
    fin = torch.zeros(B, K, dtype=torch.bool)
    fin_len = torch.zeros(B, K, dtype=torch.long)                    # generated tokens of each finished hypothesis
    unsat = torch.ones(B, 1, dtype=torch.bool)
    cur_len = P
    min_gap = float("inf")
    while True:
        flat = running[:, :, :cur_len].reshape(BK, cur_len)
        lp = pr(flat, F.log_softmax(logits.float(), dim=-1))
        r = select_step(lp, running, run_scores, seqs, beam_scores, fin, fin_len, unsat, cur_len, P, K, eos, max_length)
        for bb in range(B):
            min_gap = min(min_gap, _adjacent_gap(r["topv"][bb:bb + 1, :K + 1]),
                          _adjacent_gap(r["topv"][bb:bb + 1][:, ~r["hits"][bb]][:, :K + 1]))
        running, run_scores, parent, hits = r["running"], r["run_scores"], r["parent"], r["hits"]
        seqs, beam_scores, fin, fin_len = r["seqs"], r["beam_scores"], r["fin"], r["fin_len"]
        # cache reorder
        beam_idx = (parent + torch.arange(B)[:, None] * K).reshape(BK)
        src = beam_idx.repeat(2) if use_cfg else beam_idx
        for i in range(cfg.decoder_layers):
            st.k[i] = st.k[i].index_select(0, src)
            st.v[i] = st.v[i].index_select(0, src)
        cur_len += 1
        best_running = run_scores[:, :1] / float((cur_len - P) ** 1.0)
        worst_fin = torch.where(fin, beam_scores.min(dim=1, keepdim=True).values, torch.tensor(-1.0e9))
        unsat = unsat & torch.any(best_running > worst_fin, dim=-1, keepdim=True)
        if not (bool(unsat.any()) and not bool(hits.all())):
            break
        step_ids = running[:, :, cur_len - 1].reshape(BK, 1)
        if use_cfg:
            step_ids = step_ids.repeat(2, 1)
        logits = W.decoder_forward(st, step_ids, None, position_rule)[:, -1]
    elapsed = time.perf_counter() - t0
    gen_len = torch.where(fin[:, 0], fin_len[:, 0], torch.zeros_like(fin_len[:, 0]))
    out = seqs[:, 0, :P + int(gen_len.max())]
    prompt_counts = mask.long().sum(-1)
    out_counts = out.ne(pad_id).long().sum(-1)
    gen_counts = torch.clamp(out_counts - prompt_counts, min=0)
    n = int(gen_counts.sum())
    stats = {"generated_tokens": n, "generated_tokens_per_sample": gen_counts.tolist(),
             "elapsed_seconds": float(elapsed), "tokens_per_second": n / elapsed if elapsed > 0 else 0.0}
    return out, stats, beam_scores[:, 0].clone(), min_gap


def beam_cases():
    """name -> (prompt, negative_prompt, generate_kwargs, pcm_seed) for the beam fixtures (tests/golden/beam_reference.npz):
    every `cases.generate_cases()` prompt at K = 2 and 4, a batch whose rows finish at different lengths, `long_P150` at K = 2,
    and a timing-pre-pass-shaped call (timing context, B = 4, top_k = 50 passed, timing temperature != temperature)."""
    from . import cases
    out = {}
    for name, (prompt, neg, gk, seed) in cases.generate_cases().items():
        for K in (2, 4):
            out[f"{name}_K{K}"] = (prompt, neg, dict(gk, num_beams=K), seed)
    out["b2_filler_K2"] = (torch.tensor([[3700, 3705, 1, 9, 3645, 30], [3701, 3706, 1, 9, 3650, 12]]), None,
                           dict(GK_BEAM, num_beams=2, max_length=64, lookback_time=4092.0, lookahead_time=3273.6, context_type="map"), 4)
    prompt, gk, seed = cases.long_context_cases()["long_P150"]
    out["long_P150_K2"] = (prompt, None, dict(gk, num_beams=2), seed)
    timing = torch.tensor([[3700, 1, 5, 3650, 20], [3701, 1, 5, 3652, 70], [3702, 1, 5, 3651, 40], [3703, 1, 5, 3653, 15]])
    out["timing_prepass_B4_K2"] = (timing, None, dict(GK_BEAM, num_beams=2, top_k=50, timing_temperature=0.3, max_length=5 + 24,
                                                      lookback_time=0.0, lookahead_time=0.0, context_type="timing"), 31)
    return out
