"""Ragged batched generate on the GPU: N independent requests (own prompt length, window kind, stop set, temperatures, seed) in one
token loop through `mb200_model_generate_ragged`, each row bit-identical in its ids to the batch-1 call of that request — against
the unmodified reference (tests/golden/ragged_reference.npz, which tests/test_oracle_ragged.py pins the CPU oracle to) and against
the engine's own batch-1 `generate()` under both of its token-loop drivers."""
import os

import numpy as np
import pytest
import torch

from oracle import beam, cases, ragged

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


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


def _first_divergence(got: np.ndarray, want: np.ndarray):
    n = min(got.shape[1], want.shape[1])
    bad = np.flatnonzero(got[0, :n] != want[0, :n])
    if bad.size:
        t = int(bad[0])
        return f"position {t}: got {int(got[0, t])}, want {int(want[0, t])}"
    return f"shapes {got.shape} vs {want.shape}"


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and np.array_equal(got, want), f"{what}: {_first_divergence(got, want)}"


def _encode(model, cfg, reqs, slot_begin=0):
    model.engine.encode(torch.cat([cases.model_pcm(cfg, 1, q["seed"]) for q in reqs]).cuda(), slot_begin=slot_begin)


def _engine_requests(reqs, slot_begin=0):
    return [(slot_begin + r, q["prompt"][0], dict(q["gk"]), None if q["neg"] is None else q["neg"][0]) for r, q in enumerate(reqs)]


def _single(model, layout, slot, q, mega):
    model.engine.set_option("mega", mega)
    try:
        return model.engine.generate([slot], q["prompt"], None, layout, dict(q["gk"]), negative_prompt=q["neg"])
    finally:
        model.engine.set_option("mega", 2)


@pytest.mark.parametrize("case", list(ragged.ragged_cases()))
def test_ragged_equals_reference_and_batch1_calls(tiny16, layout, gold, case):
    from mapperatorinator_b200.server import model_generate_requests
    cfg, sd, model = tiny16
    reqs = ragged.ragged_cases()[case]
    out = model_generate_requests(model, layout, [(ragged.model_kwargs(cfg, q), dict(q["gk"])) for q in reqs])
    for r, (q, (ids, stats)) in enumerate(zip(reqs, out)):
        _same(ids.numpy(), gold[f"{case}/{r}/ids"], f"{case}[{r}] vs reference")
        assert stats["generated_tokens_per_sample"] == gold[f"{case}/{r}/counts"].tolist()
    _encode(model, cfg, reqs)
    for r, q in enumerate(reqs):
        for mega in (2, 0):
            _same(_single(model, layout, r, q, mega).numpy(), out[r][0].numpy(), f"{case}[{r}] batch-1 call, mega={mega}")


def test_order_and_neighbours_do_not_matter(tiny16, layout, gold):
    """The same requests permuted give the same per-request ids, and a request decoded beside 1, 3 and 15 other rows gives the ids it
    gives alone."""
    cfg, sd, model = tiny16
    cs = ragged.ragged_cases()
    pool = cs["mixed_windows"] + cs["mixed_stops"] + cs["mixed_temperature"]
    pool = (pool + pool)[:16]
    _encode(model, cfg, pool)
    er = _engine_requests(pool)
    want = [gold[f"{c}/{r}/ids"] for c in ("mixed_windows", "mixed_stops", "mixed_temperature") for r in range(len(cs[c]))]
    want = (want + want)[:16]
    perm = [5, 2, 9, 0, 7, 3, 10, 1, 8, 6, 4]
    for got, k in zip(model.engine.generate_ragged([er[k] for k in perm], layout), perm):
        _same(got.numpy(), want[k], f"permuted, request {k}")
    for n in (1, 2, 4, 16):
        got = model.engine.generate_ragged(er[3:4] + er[4:3 + n] if n < 16 else er[3:] + er[:3], layout)
        _same(got[0].numpy(), want[3], f"request 3 beside {n - 1} other rows")
    for k, got in enumerate(model.engine.generate_ragged(er, layout)):
        _same(got.numpy(), want[k], f"16 rows, request {k}")


def test_sampling_uses_each_requests_seed_and_temperature(tiny16, layout):
    """do_sample with top_p 0.9 and an explicit seed per request: the draws of a ragged row are those of its batch-1 call with that
    seed (row index 0 in the counter), whose temperature is decided on the row's own last tokens (request 0 ends on a beat type ->
    timing temperature; request 1 does not); two rows with the same request and seed draw the same stream."""
    cfg, sd, model = tiny16
    base = ragged.ragged_cases()["mixed_temperature"]
    reqs = []
    for k, q in enumerate(base + base[:1]):
        gk = dict(q["gk"], do_sample=True, top_p=0.9, seed=[1234, 99, 7, 1234][k], timing_temperature=0.3, temperature=[1.0, 1.3, 0.8, 1.0][k])
        reqs.append(dict(q, gk=gk))
    _encode(model, cfg, reqs)
    got = model.engine.generate_ragged(_engine_requests(reqs), layout)
    for r, q in enumerate(reqs):
        for mega in (2, 0):
            _same(got[r].numpy(), _single(model, layout, r, q, mega).numpy(), f"sampled request {r}, mega={mega}")
    assert torch.equal(got[0], got[3])


def test_uniform_and_beam_calls_after_a_ragged_call(tiny16, layout):
    """A ragged call with 4 decoder rows, then a uniform CFG call (B = 2, 4 rows) on the graph path and a beam call (B = 2, K = 2,
    4 rows) on the same engine: neither may replay the ragged token-step graph."""
    from mapperatorinator_b200.server import model_generate
    cfg, sd, model = tiny16
    reqs = ragged.ragged_cases()["mixed_windows"]
    _encode(model, cfg, reqs)
    model.engine.generate_ragged(_engine_requests(reqs), layout)

    def mk(prompt, neg, seed):
        return dict(inputs=cases.model_pcm(cfg, prompt.shape[0], seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0),
                    negative_prompt=neg, negative_prompt_attention_mask=None if neg is None else neg.ne(0))
    prompt, neg, gk, seed = cases.generate_cases()["b2_cfg"]
    model.engine.set_option("mega", 0)
    try:
        got, _ = model_generate(model, layout, mk(prompt, neg, seed), dict(gk))
    finally:
        model.engine.set_option("mega", 2)
    want = np.load(os.path.join(GOLDEN, "generate_reference.npz"))["torchaudio/b2_cfg/ids"]
    assert np.array_equal(got.numpy(), want)
    prompt, neg, gk, seed = beam.beam_cases()["b2_leftpad_lookback_K2"]
    got, _ = model_generate(model, layout, mk(prompt, neg, seed), dict(gk))
    assert np.array_equal(got.numpy(), np.load(os.path.join(GOLDEN, "beam_reference.npz"))["b2_leftpad_lookback_K2/ids"])


def test_rejected_calls_launch_nothing_and_leave_the_engine_usable(tiny16, layout, gold):
    from mapperatorinator_b200 import _lib
    cfg, sd, model = tiny16
    cs = ragged.ragged_cases()
    _encode(model, cfg, cs["mixed_windows"])
    plain, guided = _engine_requests(cs["mixed_windows"]), _engine_requests(cs["cfg_all"])
    lib = _lib.load()
    before = lib.mb200_launch_count()
    with pytest.raises(ValueError, match="classifier-free guidance"):
        model.engine.generate_ragged([plain[0], guided[0]], layout)
    with pytest.raises(ValueError, match="beam"):
        model.engine.generate_ragged([plain[0], (1, plain[1][1], dict(plain[1][2], num_beams=2), None)], layout)
    with pytest.raises(ValueError, match="max_length"):
        model.engine.generate_ragged([plain[0], (1, plain[1][1], dict(plain[1][2], max_length=9), None)], layout)
    with pytest.raises(ValueError, match="max_batch"):
        model.engine.generate_ragged([plain[k % 4] for k in range(17)], layout)
    with pytest.raises(ValueError, match="max_batch"):
        model.engine.generate_ragged([guided[k % 2] for k in range(9)], layout)
    assert lib.mb200_launch_count() == before
    for r, got in enumerate(model.engine.generate_ragged(plain, layout)):
        _same(got.numpy(), gold[f"mixed_windows/{r}/ids"], f"after the rejected calls, request {r}")


def test_decode_songs_ragged_equals_decode_windows_per_song(tiny16, layout):
    """3 songs of 4 / 2 / 3 windows, look-back prompts built from what the previous window generated (`trim_predicted_tokens`), so
    prompt lengths differ per song and step; first and last windows of different songs share a step."""
    from mapperatorinator_b200.pipeline import SongDecoder, trim_predicted_tokens
    cfg, sd, model = tiny16
    counts, stride = [4, 2, 3], 4
    model.engine.encode(torch.cat([cases.model_pcm(cfg, 1, 100 + k) for k in range(12)]).cuda(), slot_begin=0)
    head = [[3700, 3705, 1, 9], [3701, 3706, 3711, 1, 9], [3702, 1, 9]]
    lb_ms, la_ms = 4092.0, 3273.6

    def prompt_fn(s, i, streams):
        if i == 0:
            return head[s]
        return head[s] + trim_predicted_tokens(streams[i - 1], layout, "map", lb_ms, 8184.0 - la_ms, trim_lookahead=True)[-(20 + 3 * s):]

    def gk_fn(s, i):
        return dict(cases.GK, max_length=64 + 8 * s, min_new_tokens=6 + 5 * s + i, lookback_time=lb_ms if i > 0 else 0.0,
                    lookahead_time=la_ms if i < counts[s] - 1 else 0.0, context_type="map")
    song = SongDecoder(model, layout)
    got = song.decode_songs_ragged(counts, prompt_fn, gk_fn, windows_per_song=stride)
    lengths = set()
    for s, n in enumerate(counts):
        want = song.decode_windows(n, lambda i, st, s=s: prompt_fn(s, i, st), lambda i, s=s: gk_fn(s, i), slot_begin=s * stride)
        assert got[s] == want, f"song {s}"
        lengths.update((i, len(prompt_fn(s, i, want))) for i in range(1, n))
    assert len({p for i, p in lengths if i == 1}) > 1


def _full_requests(n, new=64):
    """n requests with prompt lengths spread over 17..600 (the last one: max_length 664, 11 self-attention splits), then two at the
    model's long plans: max_length 1025 (17 splits) and 2048 (32 splits, the reference's own max_length)."""
    g = torch.Generator().manual_seed(n)
    lens = torch.linspace(17, 600, n).round().long().tolist() + [1025 - new, 2048 - new]
    reqs = []
    for r, P in enumerate(lens):
        prompt = torch.randint(17, 3600, (1, P), generator=g)
        prompt[0, :4] = torch.tensor([3700, 3705, 1, 9])
        gk = dict(cases.GK, max_length=P + new, min_new_tokens=new, lookback_time=4092.0 if r % 2 else 0.0, lookahead_time=3273.6 if r % 3 else 0.0,
                  context_type="map")
        reqs.append(dict(prompt=prompt, neg=None, gk=gk, seed=r))
    return reqs


def test_ragged_equals_batch1_calls_full_dims(layout):
    """whisper-small dimensions: 9 and 18 requests with prompt lengths spread over 17..600 plus max_length 1025 and 2048 on resident
    encoder slots, 64 tokens each, equal their batch-1 calls on the default driver."""
    from mapperatorinator_b200 import v29_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = v29_model_config()
    model = B200Mapperatorinator(cfg, init_model_state_dict(cfg, 0), max_windows=18, max_batch=18)
    reqs = _full_requests(16)
    n = len(reqs)
    assert [q["gk"]["max_length"] for q in reqs[-3:]] == [664, 1025, 2048]
    model.engine.encode(torch.cat([cases.model_pcm(cfg, 1, q["seed"]) for q in reqs]).cuda(), slot_begin=0)
    er = _engine_requests(reqs)
    want = [_single(model, layout, r, q, 2) for r, q in enumerate(reqs)]
    for pick in (list(range(0, n, 2)), list(range(n))):
        for k, got in zip(pick, model.engine.generate_ragged([er[k] for k in pick], layout)):
            assert got.shape[1] == reqs[k]["prompt"].shape[1] + 64
            _same(got.numpy(), want[k].numpy(), f"{len(pick)} requests, request {k} (P = {reqs[k]['prompt'].shape[1]})")
