"""Drop-in for the model-call boundary of the reference: `osuT5.osuT5.inference.server.model_generate` / `model_forward`
(osuT5/osuT5/inference/server.py:72-181).  Same signature, same returns (CPU LongTensor of prompt+generated ids, stats dict
with the reference's token accounting, :50-69), so `Processor.model_generate` (processor.py:155-176) can call it unchanged
with a `B200Mapperatorinator` as `model`.
"""
from __future__ import annotations

import time

import torch

from .token_layout import TokenLayout


def get_eos_token_id(tokenizer, lookback_time: float = 0, lookahead_time: float = 0, context_type=None):
    """server.py:72-80."""
    return TokenLayout.from_tokenizer(tokenizer).eos_token_ids(lookback_time, lookahead_time, context_type)


def _build_generation_stats(result: torch.Tensor, model_kwargs: dict, pad_token_id, elapsed_seconds: float) -> dict:
    """server.py:50-69: generated = non-pad output tokens minus non-pad prompt tokens, per row, clamped at 0."""
    mask = model_kwargs.get("decoder_attention_mask")
    ids = model_kwargs.get("decoder_input_ids")
    if isinstance(mask, torch.Tensor):
        prompt_counts = mask.to(torch.long).sum(dim=-1).cpu()
    elif pad_token_id is None:
        prompt_counts = torch.full((ids.shape[0],), ids.shape[1], dtype=torch.long)
    else:
        prompt_counts = ids.ne(pad_token_id).to(torch.long).sum(dim=-1).cpu()
    if pad_token_id is None:
        out_counts = torch.full((result.shape[0],), result.shape[1], dtype=torch.long)
    else:
        out_counts = result.ne(pad_token_id).to(torch.long).sum(dim=-1)
    gen = torch.clamp(out_counts - prompt_counts, min=0)
    n = int(gen.sum().item())
    return {"generated_tokens": n, "generated_tokens_per_sample": gen.tolist(), "elapsed_seconds": float(elapsed_seconds),
            "tokens_per_second": n / elapsed_seconds if elapsed_seconds > 0 else 0.0}


@torch.no_grad()
def model_generate(model, tokenizer, model_kwargs, generate_kwargs):
    """`model_generate(model, tokenizer, model_kwargs, generate_kwargs) -> (LongTensor[B, P+N] on CPU, stats)`.
    `precision` is accepted for signature parity and ignored: the engine computes in fp32 (the parity contract of the hot path), and
    `precision='amp'` stays fp32.  The model's LOAD precision decides the weight store: a model loaded in bf16 (every decoder GEMV
    matrix and proj_out bf16) has its token loop's per-kernel GEMVs read a bf16 copy of those weights, with the same ids as the same
    values served from fp32 (`ModelEngine.token_weight_dtype`)."""
    generate_kwargs = dict(generate_kwargs)
    generate_kwargs.pop("precision", None)
    layout = TokenLayout.from_tokenizer(tokenizer)
    pad_token_id = generate_kwargs.get("pad_token_id", getattr(tokenizer, "pad_id", None))
    start = time.perf_counter()
    result = model.generate(
        inputs=model_kwargs["inputs"], decoder_input_ids=model_kwargs["decoder_input_ids"],
        decoder_attention_mask=model_kwargs.get("decoder_attention_mask"), negative_prompt=model_kwargs.get("negative_prompt"),
        negative_prompt_attention_mask=model_kwargs.get("negative_prompt_attention_mask"), tokenizer=layout,
        generate_kwargs=generate_kwargs)
    elapsed = time.perf_counter() - start
    result = result.cpu()
    return result, _build_generation_stats(result, model_kwargs, pad_token_id, elapsed)


@torch.no_grad()
def model_generate_requests(model, tokenizer, requests):
    """Several independent `model_generate` calls of batch size 1 in ONE token loop (what `Processor.generate_sequential` issues one
    after another, and what `InferenceServer._batch_thread` packs from several clients).  `requests` is a list of
    `(model_kwargs, generate_kwargs)` with batch-1 tensors and no padding; the result is a list of `(ids, stats)` equal, request by
    request, to `model_generate(model, tokenizer, model_kwargs, generate_kwargs)`; `elapsed_seconds` is the shared call's."""
    layout = TokenLayout.from_tokenizer(tokenizer)
    n = len(requests)
    if n > model.engine.max_windows:
        raise ValueError(f"{n} requests need {n} encoder slots; this engine was built with max_windows={model.engine.max_windows}")
    reqs = [(r, *_batch1_request(mk, gk)) for r, (mk, gk) in enumerate(requests)]
    start = time.perf_counter()
    model.engine.encode(torch.cat([mk["inputs"] for mk, _ in requests]).to(model.device, torch.float32), slot_begin=0)
    results = model.engine.generate_ragged(reqs, layout)
    elapsed = time.perf_counter() - start
    out = []
    for (mk, gk), res in zip(requests, results):
        pad_token_id = gk.get("pad_token_id", getattr(tokenizer, "pad_id", None))
        out.append((res, _build_generation_stats(res, mk, pad_token_id, elapsed)))
    return out


def _batch1_request(mk: dict, gk: dict):
    """The rules of a request of a ragged call or stream: batch 1, prompt without padding -> (prompt ids, kwargs, negative prompt)."""
    gk = dict(gk)
    gk.pop("precision", None)
    ids = mk["decoder_input_ids"]
    if ids.shape[0] != 1 or mk["inputs"].shape[0] != 1:
        raise ValueError("every request of a ragged call is a batch-1 call")
    mask = mk.get("decoder_attention_mask")
    if isinstance(mask, torch.Tensor) and not bool(mask.all()):
        raise ValueError("a request of a ragged call carries its prompt without padding")
    neg = mk.get("negative_prompt")
    return ids[0], gk, None if neg is None else neg[0]


@torch.no_grad()
def model_generate_stream(model, tokenizer, requests, max_rows=None):
    """Continuous batching: the batch-1 `(model_kwargs, generate_kwargs)` of `requests` (the rules of `model_generate_requests`) go
    through one decode stream of `max_rows` rows.  `requests` is any iterable, read one request ahead as rows free up; an item `None`
    means "nothing ready yet" (a server's queue that is momentarily empty) and is skipped without waiting.  Requests are admitted in
    order as soon as a row is free, each into the encoder slot of its row (the frames of one poll's admissions are encoded as one
    chunk per run of adjacent slots), and yielded as `(index, ids, stats)` in the order they finish, `index` counting the requests;
    `(ids, stats)` is what `model_generate` returns for that request, with `elapsed_seconds` from its admission to its hand-back.
    Every request is guided (negative prompt, cfg_scale > 1) or none is, as the first request is."""
    layout = TokenLayout.from_tokenizer(tokenizer)
    engine = model.engine
    it = iter(requests)
    end = object()
    count = 0

    def pull():
        """(index, model_kwargs, generate_kwargs), None when nothing is ready, `end` when the iterable is exhausted."""
        nonlocal count
        item = next(it, end)
        if item is end or item is None:
            return item
        count += 1
        return (count - 1, *item)
    pending = pull()
    while pending is None:
        pending = pull()
    if pending is end:
        return
    _, first_mk, first_gk = pending
    guided = first_mk.get("negative_prompt") is not None and float(first_gk.get("cfg_scale", 1.0)) > 1.0
    per = 2 if guided else 1
    limit = min(engine.max_windows, engine.max_batch // per)
    if max_rows is None:
        max_rows = limit
    if not 1 <= max_rows <= limit:
        raise ValueError(f"max_rows={max_rows}: a row needs its own encoder slot and {per} decoder row(s); this engine allows "
                         f"1..{limit} (max_windows={engine.max_windows}, max_batch={engine.max_batch})")
    live = {}            # row -> (index, model_kwargs, generate_kwargs, admission time)
    with engine.open_stream(layout, max_rows, guidance=guided) as stream:
        while True:
            free = [r for r in range(max_rows) if r not in live]     # the stream fills its lowest free rows first
            batch = []
            while pending is not end:
                if pending is None:
                    pending = pull()
                    if pending is None:
                        break
                    continue
                if len(batch) == len(free):
                    break                                            # `pending` waits for the next free row
                idx, mk, gk = pending
                prompt, gk, neg = _batch1_request(mk, gk)
                batch.append((free[len(batch)], idx, mk, gk, prompt, neg))
                pending = None
            if batch:
                k = 0
                while k < len(batch):          # adjacent slots in one encoder chunk
                    j = k + 1
                    while j < len(batch) and batch[j][0] == batch[j - 1][0] + 1:
                        j += 1
                    engine.encode(torch.cat([b[2]["inputs"] for b in batch[k:j]]).to(model.device, torch.float32), slot_begin=batch[k][0])
                    k = j
                for row, idx, mk, gk, prompt, neg in batch:
                    got = stream.admit(row, prompt, gk, negative_prompt=neg)
                    assert got == row, (got, row)
                    live[row] = (idx, mk, gk, time.perf_counter())
            if not live:
                if pending is end:
                    return
                continue
            for row, ids in stream.run(waiting=0 if pending is None or pending is end else 1):
                idx, mk, gk, t0 = live.pop(row)
                pad_token_id = gk.get("pad_token_id", getattr(tokenizer, "pad_id", None))
                yield idx, ids, _build_generation_stats(ids, mk, pad_token_id, time.perf_counter() - t0)


@torch.no_grad()
def model_forward(model, model_kwargs, generate_kwargs):
    """server.py:159-181 (cfg_scale == 1 path): teacher-forced fp32 logits on the CPU."""
    out = model.forward(frames=model_kwargs["inputs"], decoder_input_ids=model_kwargs["decoder_input_ids"],
                        decoder_attention_mask=model_kwargs.get("decoder_attention_mask"))
    return out.logits.to(torch.float32).cpu()


@torch.no_grad()
def model_score(model, model_kwargs, generate_kwargs):
    """MaiMod's scoring of given tokens (processor.py:511-525) on the teacher-forced pass `model_forward` runs, reduced on the
    device: takes `model_forward`'s arguments and returns a dict of CPU tensors [B, L] indexed by the scored token (`entropy`,
    `surprisal`, `relative`, `suggested`; see `ModelEngine.score_tokens`), so the caller slices `[start + padding, end + padding)`
    where it sliced the logits at `[start + padding - 1, end + padding - 1)`.  `precision` is accepted and ignored (fp32); the
    teacher-forced pass reads the fp32 weights whatever precision the model was loaded in.
    A guided call (`cfg_scale > 1` with a negative prompt) is refused: the reference repeats the decoder rows but not the frames
    there, which is not a pass worth mirroring."""
    generate_kwargs = dict(generate_kwargs)
    generate_kwargs.pop("precision", None)
    if generate_kwargs.get("cfg_scale", 1.0) > 1.0 and model_kwargs.get("negative_prompt") is not None:
        raise ValueError("model_score does not run a guided (cfg_scale > 1, negative prompt) teacher-forced pass")
    out = model.score(frames=model_kwargs["inputs"], decoder_input_ids=model_kwargs["decoder_input_ids"],
                      decoder_attention_mask=model_kwargs.get("decoder_attention_mask"))
    return {k: v.cpu() for k, v in out.items()}
