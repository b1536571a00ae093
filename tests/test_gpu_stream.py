"""Decode stream (continuous batching) on the GPU: requests admitted into the free rows of a running ragged token loop, handed back as
they finish, their rows reused — every request's ids equal to its own batch-1 call, whatever step it joins at, whatever its neighbours
do and whatever its row held before.  Against the unmodified reference (tests/golden/ragged_reference.npz: a stream row is a batch-1
call) and against the engine's own batch-1 `generate()` under both of its token-loop drivers."""
import os
from collections import deque

import numpy as np
import pytest
import torch

from oracle import cases, ragged

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LB, LA = ragged.LB, ragged.LA


@pytest.fixture(scope="module")
def tiny16():
    from mapperatorinator_b200 import tiny_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd = init_model_state_dict(cfg, 0)
    return cfg, sd, B200Mapperatorinator(cfg, sd, max_windows=24, max_batch=16)


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "ragged_reference.npz"))


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    n = min(got.shape[-1], want.shape[-1])
    bad = np.flatnonzero(got.reshape(-1)[:n] != want.reshape(-1)[:n])
    where = f"position {int(bad[0])}" if bad.size else f"shapes {got.shape} vs {want.shape}"
    assert got.shape == want.shape and np.array_equal(got, want), f"{what}: {where}"


def _single(model, layout, slot, q, mega):
    model.engine.set_option("mega", mega)
    try:
        return model.engine.generate([slot], q["prompt"], None, layout, dict(q["gk"]), negative_prompt=q["neg"])
    finally:
        model.engine.set_option("mega", 2)


def _encode(model, cfg, reqs, slot_begin=0):
    model.engine.encode(torch.cat([cases.model_pcm(cfg, 1, q["seed"]) for q in reqs]).cuda(), slot_begin=slot_begin)


def _admit(stream, slot, q):
    return stream.admit(slot, q["prompt"][0], dict(q["gk"]), None if q["neg"] is None else q["neg"][0])


def _req(P, seed, **gk):
    return dict(prompt=ragged._prompt(P, seed), neg=None, gk=dict(cases.GK, **gk), seed=seed)


def _drain(stream, got, rows, waiting=0):
    """run() until every live row has been handed back; got[request] = ids, rows[row] -> request."""
    while stream.live_rows:
        for row, ids in stream.run(waiting=waiting):
            got[rows.pop(row)] = ids


@pytest.mark.parametrize("case", list(ragged.ragged_cases()))
def test_stream_equals_reference_with_queued_requests(tiny16, layout, gold, case):
    """Every case of the ragged reference through `model_generate_stream` with fewer rows than requests, so requests queue and rows
    are reused, from a source that is not always ready; each request's ids and token count equal the reference's batch-1 call."""
    from mapperatorinator_b200.server import model_generate_stream
    cfg, sd, model = tiny16
    reqs = ragged.ragged_cases()[case]
    seen = set()
    # a `None` between requests: a source with nothing ready at that poll
    source = (item for q in reqs for item in (None, (ragged.model_kwargs(cfg, q), dict(q["gk"]))))
    for idx, ids, stats in model_generate_stream(model, layout, source, max_rows=max(1, len(reqs) - 2)):
        _same(ids.numpy(), gold[f"{case}/{idx}/ids"], f"{case}[{idx}] vs reference")
        assert stats["generated_tokens_per_sample"] == gold[f"{case}/{idx}/counts"].tolist()
        assert stats["elapsed_seconds"] > 0
        seen.add(idx)
    assert seen == set(range(len(reqs)))


def test_arrival_at_any_step(tiny16, layout):
    """The same request admitted when its neighbour has made 0, 1, 17 selections, and when the neighbour's next key crosses the
    128-key split boundary, gives the ids of its batch-1 call under both drivers.  Greedy, look-back bias on, min_new_tokens,
    time-shift bias, conditional temperature (mixed_temperature: one request ends on a beat type, the other does not)."""
    cfg, sd, model = tiny16
    targets = ragged.ragged_cases()["mixed_temperature"][:2]
    # neighbour: P 100, min_new_tokens 28 -> the first burst (stretched to its earliest stop) leaves it at cur_len 128
    neighbours = {1: _req(40, 61, max_length=200, lookback_time=LB, lookahead_time=LA, context_type="map"),
                  17: _req(40, 62, max_length=200, min_new_tokens=17, lookback_time=LB, lookahead_time=LA, context_type="map"),
                  28: _req(100, 63, max_length=300, min_new_tokens=28, lookback_time=LB, lookahead_time=LA, context_type="map")}
    _encode(model, cfg, targets + list(neighbours.values()))          # slots 0, 1: targets; 2, 3, 4: neighbours
    want = [[_single(model, layout, t, q, mega) for mega in (2, 0)] for t, q in enumerate(targets)]
    for t, q in enumerate(targets):
        _same(want[t][0].numpy(), want[t][1].numpy(), f"target {t}: the two drivers")
        for arrival in (0, 1, 17, 28):
            got, rows = {}, {}
            with model.engine.open_stream(layout, 2) as stream:
                if arrival == 0:
                    rows[_admit(stream, t, q)] = "target"
                    rows[_admit(stream, 2, neighbours[1])] = "neighbour"
                else:
                    nb = neighbours[arrival]
                    rows[_admit(stream, 2 + list(neighbours).index(arrival), nb)] = "neighbour"
                    if arrival > 1:
                        for row, ids in stream.run(waiting=1):
                            got[rows.pop(row)] = ids
                        assert "neighbour" not in got, f"arrival {arrival}: the neighbour stopped before the target joined"
                    rows[_admit(stream, t, q)] = "target"
                _drain(stream, got, rows)
            _same(got["target"].numpy(), want[t][0].numpy(), f"target {t} admitted at neighbour step {arrival}")


def test_sampling_admitted_mid_stream(tiny16, layout):
    """do_sample with top_p and an explicit seed per request, admitted while another sampled request runs: the counter-based draws
    are those of the batch-1 call with that seed."""
    cfg, sd, model = tiny16
    base = ragged.ragged_cases()["mixed_temperature"]
    reqs = [dict(q, gk=dict(q["gk"], do_sample=True, top_p=0.9, seed=s, timing_temperature=0.3)) for q, s in zip(base, (1234, 99, 7))]
    _encode(model, cfg, reqs)
    got, rows = {}, {}
    with model.engine.open_stream(layout, 3) as stream:
        rows[_admit(stream, 0, reqs[0])] = 0
        for k in (1, 2):
            for row, ids in stream.run(waiting=1):
                got[rows.pop(row)] = ids
            rows[_admit(stream, k, reqs[k])] = k
        _drain(stream, got, rows)
    for k, q in enumerate(reqs):
        for mega in (2, 0):
            _same(got[k].numpy(), _single(model, layout, k, q, mega).numpy(), f"sampled request {k}, mega={mega}")


def test_row_reuse_leaks_nothing(tiny16, layout):
    """One row: a 600-token request, then a 17-token one in the same row, and the reverse order.  Both equal their batch-1 calls,
    so no stale key, look-back score or time-shift state of the row's previous request leaks."""
    cfg, sd, model = tiny16
    long_q = _req(40, 71, max_length=640, min_new_tokens=600, lookback_time=LB, lookahead_time=LA, context_type="map")
    short_q = _req(12, 72, max_length=12 + 17, min_new_tokens=17, lookback_time=LB, lookahead_time=LA, context_type="map",
                   timeshift_bias=0.5)
    _encode(model, cfg, [long_q, short_q])
    want = [_single(model, layout, k, q, 2) for k, q in enumerate((long_q, short_q))]
    assert want[0].shape[1] == 640 and want[1].shape[1] == 29
    for order in ((0, 1), (1, 0)):
        with model.engine.open_stream(layout, 1) as stream:
            for k in order:
                got, rows = {}, {}
                rows[_admit(stream, k, (long_q, short_q)[k])] = k
                assert list(rows) == [0]
                _drain(stream, got, rows)
                _same(got[k].numpy(), want[k].numpy(), f"request {k} in order {order}")


def test_live_row_untouched_by_admissions(tiny16, layout):
    """A long request runs while 15 others are admitted and handed back around it through the stream's other 3 rows."""
    cfg, sd, model = tiny16
    long_q = _req(30, 80, max_length=330, min_new_tokens=300, lookback_time=LB, lookahead_time=LA, context_type="map")
    cs = ragged.ragged_cases()
    others = (cs["mixed_windows"] + cs["mixed_stops"] + cs["mixed_temperature"]) * 2
    others = others[:15]
    _encode(model, cfg, [long_q])
    _encode(model, cfg, others, slot_begin=1)
    want_long = _single(model, layout, 0, long_q, 2)
    got, rows = {}, {}
    queue = deque(range(15))
    with model.engine.open_stream(layout, 4) as stream:
        rows[_admit(stream, 0, long_q)] = "long"
        while queue or stream.live_rows:
            while queue and stream.free_rows:
                k = queue.popleft()
                rows[_admit(stream, 1 + k, others[k])] = k
            for row, ids in stream.run(waiting=len(queue)):
                got[rows.pop(row)] = ids
    _same(got["long"].numpy(), want_long.numpy(), "the long request")
    for k, q in enumerate(others):
        _same(got[k].numpy(), _single(model, layout, 1 + k, q, 2).numpy(), f"request {k}")


def test_decode_songs_continuous(tiny16, layout):
    """3 songs of 4 / 2 / 3 windows with look-back prompts built from the previous window: `decode_songs_continuous` equals
    `decode_windows` per song and what `decode_songs_ragged` returns."""
    from mapperatorinator_b200.pipeline import SongDecoder, trim_predicted_tokens
    cfg, sd, model = tiny16
    counts, stride = [4, 2, 3], 4
    model.engine.encode(torch.cat([cases.model_pcm(cfg, 1, 100 + k) for k in range(12)]).cuda(), slot_begin=0)
    head = [[3700, 3705, 1, 9], [3701, 3706, 3711, 1, 9], [3702, 1, 9]]

    def prompt_fn(s, i, streams):
        if i == 0:
            return head[s]
        return head[s] + trim_predicted_tokens(streams[i - 1], layout, "map", LB, 8184.0 - LA, trim_lookahead=True)[-(20 + 3 * s):]

    def gk_fn(s, i):
        return dict(cases.GK, max_length=64 + 8 * s, min_new_tokens=6 + 5 * s + i, lookback_time=LB if i > 0 else 0.0,
                    lookahead_time=LA if i < counts[s] - 1 else 0.0, context_type="map" if s != 1 else "kiai")
    song = SongDecoder(model, layout)
    got = song.decode_songs_continuous(counts, prompt_fn, gk_fn, windows_per_song=stride)
    assert got == song.decode_songs_ragged(counts, prompt_fn, gk_fn, windows_per_song=stride)
    for s, n in enumerate(counts):
        want = song.decode_windows(n, lambda i, st, s=s: prompt_fn(s, i, st), lambda i, s=s: gk_fn(s, i), slot_begin=s * stride)
        assert got[s] == want, f"song {s}"


def test_rejections_launch_nothing_and_leave_stream_and_engine_usable(tiny16, layout, gold):
    from mapperatorinator_b200 import _lib
    from mapperatorinator_b200.server import model_generate_stream
    cfg, sd, model = tiny16
    eng = model.engine
    cs = ragged.ragged_cases()
    plain, guided = cs["mixed_windows"], cs["cfg_all"]
    _encode(model, cfg, plain)
    lib = _lib.load()
    with eng.open_stream(layout, 1, max_length=64) as stream:
        row = _admit(stream, 0, plain[0])
        before = lib.mb200_launch_count()
        with pytest.raises(ValueError, match="busy"):
            _admit(stream, 1, plain[1])
        # the engine's own check, below the Python one
        params, vflags, flat, off, nflat, slots, _ = eng._ragged_args([(1, plain[1]["prompt"][0], dict(plain[1]["gk"]), None)], layout)
        rows_out = np.zeros(1, dtype=np.int32)
        assert lib.mb200_stream_admit(stream.handle, 1, slots.ctypes.data, flat.ctypes.data, off.ctypes.data, None, vflags.ctypes.data,
                                      _lib.C.cast(params, _lib.C.c_void_p), rows_out.ctypes.data, None) != 0
        assert b"free rows" in lib.mb200_last_error()
        with pytest.raises(ValueError, match="cap"):
            _admit(stream, 1, dict(plain[1], gk=dict(plain[1]["gk"], max_length=100)))
        with pytest.raises(ValueError, match="guided"):
            _admit(stream, 1, guided[0])
        with pytest.raises(ValueError, match="beam"):
            _admit(stream, 1, dict(plain[1], gk=dict(plain[1]["gk"], num_beams=2)))
        q = plain[1]
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.generate([1], q["prompt"], None, layout, dict(q["gk"]))
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.generate_ragged([(1, q["prompt"][0], dict(q["gk"]), None)], layout)
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.generate_beams([1], q["prompt"], None, layout, dict(q["gk"], num_beams=2))
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.forward_logits([1], q["prompt"], None)
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.score_tokens([1], q["prompt"], None)
        with pytest.raises(RuntimeError, match="already open"):
            eng.open_stream(layout, 1)
        # the PDL toggle would destroy the stream's step graph; the parity hooks and the step profiler write its state
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.set_option("pdl", 1)
        ids, V = q["prompt"], cfg.vocab_size_out
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.logits_chain(torch.zeros(1, V, device="cuda"), ids, ids.shape[1], layout, dict(q["gk"]))
        with pytest.raises(RuntimeError, match="decode stream is open"):
            eng.beam_step(torch.zeros(2, V, device="cuda"), ids.repeat(2, 1), torch.zeros(2), 2, ids.shape[1], layout, dict(q["gk"]))
        out_us = np.zeros(4, dtype=np.float32)
        with pytest.raises(RuntimeError, match="decode stream is open"):
            _lib.check(lib.mb200_model_profile_step(eng.handle, 1, 1, 64, 1, out_us.ctypes.data, None))
        assert lib.mb200_launch_count() == before
        got = {}
        _drain(stream, got, {row: 0})
        _same(got[0].numpy(), gold["mixed_windows/0/ids"], "the admitted request after the rejections")
        rows = {_admit(stream, 1, plain[1]): 1}
        _drain(stream, got, rows)
        _same(got[1].numpy(), gold["mixed_windows/1/ids"], "a request admitted after the rejections")
    # padded and batch-2 requests are refused by the generator before anything runs
    mk = ragged.model_kwargs(cfg, plain[0])
    padded = dict(mk, decoder_attention_mask=torch.cat([torch.zeros(1, 1, dtype=torch.bool), mk["decoder_attention_mask"][:, 1:]], 1))
    batch2 = dict(mk, decoder_input_ids=mk["decoder_input_ids"].repeat(2, 1), inputs=mk["inputs"].repeat(2, 1))
    for bad, what in ((padded, "padding"), (batch2, "batch-1")):
        before = lib.mb200_launch_count()
        with pytest.raises(ValueError, match=what):
            list(model_generate_stream(model, layout, [(bad, dict(plain[0]["gk"]))]))
        assert lib.mb200_launch_count() == before
    # closed: the engine's token-loop calls work again
    _encode(model, cfg, plain)
    for r, got in enumerate(eng.generate_ragged([(r, q["prompt"][0], dict(q["gk"]), None) for r, q in enumerate(plain)], layout)):
        _same(got.numpy(), gold[f"mixed_windows/{r}/ids"], f"ragged call after the stream closed, request {r}")
    _same(_single(model, layout, 0, plain[0], 2).numpy(), gold["mixed_windows/0/ids"], "batch-1 call after the stream closed")


def test_stream_equals_batch1_calls_full_dims(layout):
    """whisper-small dimensions: 24 requests with prompts spread over 17..600 and budgets of 16..128 new tokens, two of them running
    to the cap of 2048, through 8 rows; each equals its batch-1 call."""
    from mapperatorinator_b200 import v29_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = v29_model_config()
    model = B200Mapperatorinator(cfg, init_model_state_dict(cfg, 0), max_windows=24, max_batch=8)
    g = torch.Generator().manual_seed(24)
    lens = torch.linspace(17, 600, 24).round().long().tolist()
    budgets = torch.randint(16, 129, (24,), generator=g).tolist()
    budgets[5], budgets[20] = 2048 - lens[5], 2048 - lens[20]
    reqs = []
    for r, (P, n) in enumerate(zip(lens, budgets)):
        prompt = torch.randint(17, 3600, (1, P), generator=g)
        prompt[0, :4] = torch.tensor([3700, 3705, 1, 9])
        gk = dict(cases.GK, max_length=P + n, min_new_tokens=n, lookback_time=LB if r % 2 else 0.0, lookahead_time=LA if r % 3 else 0.0,
                  context_type="map")
        reqs.append(dict(prompt=prompt, neg=None, gk=gk, seed=r))
    _encode(model, cfg, reqs)
    want = [_single(model, layout, r, q, 2) for r, q in enumerate(reqs)]
    got, rows, queue = {}, {}, deque(range(24))
    with model.engine.open_stream(layout, 8) as stream:
        while queue or stream.live_rows:
            while queue and stream.free_rows:
                k = queue.popleft()
                rows[_admit(stream, k, reqs[k])] = k
            for row, ids in stream.run(waiting=len(queue)):
                got[rows.pop(row)] = ids
    for k in range(24):
        assert got[k].shape[1] == lens[k] + budgets[k]
        _same(got[k].numpy(), want[k].numpy(), f"request {k} (P = {lens[k]}, {budgets[k]} new tokens)")
