"""Per-token scoring of a teacher-forced pass on the device (`server.model_score`, MaiMod's processor.py:519-525):
  * against MaiMod's scores on the unmodified reference's logits (tests/golden/score_reference.npz, tiny model, prompts of 40 / 300 /
    700 real tokens left-padded to 700), within a bound derived from the teacher-forced logits tolerance;
  * against torch statistics on the engine's own `forward_logits` output of the same call, at whisper-small dimensions with B = 8
    and L up to tgt_seq_len (several projection chunks, the last one overlapping): the chunked projection changes no logit;
  * self-consistency with greedy generation; rejections; a generate call after a score call still matches its fixture.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import cases, score

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PCM_SEED = 6                  # oracle/make_score_golden.py
RTOL, ATOL = 2e-4, 2e-4       # teacher-forced logits tolerance (tests/test_gpu_model.py::test_teacher_forced_logits_left_padded)


@pytest.fixture(scope="module")
def tiny():
    from mapperatorinator_b200 import tiny_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    sd = init_model_state_dict(cfg, 0)
    return cfg, sd, B200Mapperatorinator(cfg, sd, max_windows=4, max_batch=4)


@pytest.fixture(scope="module")
def small():
    """whisper-small dimensions, room for 8 decoder rows of up to tgt_seq_len tokens over 8 resident encoder slots."""
    from mapperatorinator_b200 import v29_model_config
    from mapperatorinator_b200.modeling import B200Mapperatorinator
    from mapperatorinator_b200.weights import init_model_state_dict
    cfg = v29_model_config()
    sd = init_model_state_dict(cfg, 0)
    model = B200Mapperatorinator(cfg, sd, max_windows=8, max_batch=8)
    model.engine.encode((torch.randn(8, cfg.samples_per_window, generator=torch.Generator().manual_seed(2)) * 0.1).cuda(), 0)
    return cfg, model


def _mk(cfg, ids, mask, pcm_seed):
    return dict(inputs=cases.model_pcm(cfg, ids.shape[0], pcm_seed), decoder_input_ids=ids, decoder_attention_mask=mask)


def test_scores_match_reference_fixture(tiny):
    """A logits error of eps moves any log-softmax entry by at most 2 eps, i.e. 2 eps / ln 2 bits: the bound on surprisal, and on
    entropy (a p-weighted mean of such entries plus p log p terms of the same size).  eps is the teacher-forced logits tolerance
    RTOL |z| + ATOL at the largest logit of the call.  The argmax must be exact wherever the reference's top-2 gap exceeds 2 eps."""
    from mapperatorinator_b200.server import model_forward, model_score
    cfg, _, model = tiny
    gold = np.load(os.path.join(GOLDEN, "score_reference.npz"))
    ids, mask = torch.from_numpy(gold["ids"]), torch.from_numpy(gold["mask"])
    got = {k: v.numpy() for k, v in model_score(model, _mk(cfg, ids, mask, PCM_SEED), dict(precision="fp32")).items()}
    zmax = model_forward(model, _mk(cfg, ids, mask, PCM_SEED), dict(precision="fp32")).abs().max().item()
    eps = RTOL * zmax + ATOL
    bits = 2 * eps / math.log(2)
    for k in ("entropy", "surprisal", "relative"):
        assert got[k].shape == gold[k].shape and got[k].dtype == np.float32
        assert np.array_equal(np.isnan(got[k]), np.isnan(gold[k])), k
    for k in ("entropy", "surprisal"):
        ok = ~np.isnan(gold[k])
        err = np.abs(got[k][ok] - gold[k][ok]).max()
        assert err <= bits, (k, err, bits)
    assert (got["suggested"][:, 0] == -1).all() and got["suggested"].dtype == np.int64
    sure = ~(gold["top2_gap"] <= 2 * eps)
    assert np.array_equal(got["suggested"][sure], gold["suggested"][sure])


def _torch_scores(logits, ids):
    return score.score_from_logits(logits, ids.to(logits.device))


@pytest.mark.parametrize("L", [40, 1024, 2048])
def test_scores_equal_torch_on_engine_logits(small, L):
    """Same call, scored on the device vs torch on the engine's `forward_logits` output: B * L = 320 rows is one SIMT-projected chunk,
    8192 and 16384 rows are 3 and 6 tensor-core chunks with an overlapping last one.  If any chunk changed a logit, the argmax
    or the statistics would move."""
    cfg, model = small
    B = 8
    g = torch.Generator().manual_seed(L)
    ids = torch.randint(17, cfg.vocab_size_in, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.bool)
    for b in range(B):
        npad = (b * L) // 9                       # 0 .. 7/9 of the row left-padded
        ids[b, :npad] = 0
        mask[b, :npad] = False
    slots = list(range(B))
    logits = model.engine.forward_logits(slots, ids, mask)
    want = _torch_scores(logits, ids)
    del logits
    got = model.engine.score_tokens(slots, ids, mask)
    assert torch.equal(got["suggested"], want["suggested"])
    for k in ("entropy", "surprisal", "relative"):
        assert torch.equal(torch.isnan(got[k]), torch.isnan(want[k])), k
    tol = 1e-6                                    # the two sums run in different orders
    for k in ("entropy", "surprisal"):
        torch.testing.assert_close(got[k], want[k], rtol=tol, atol=tol, equal_nan=True)
    # relative = surprisal / entropy carries both relative errors: (tol |s| + tol) / |s| + (tol |e| + tol) / |e|
    s, e, rel = want["surprisal"], want["entropy"], want["relative"]
    ok = ~torch.isnan(rel)
    bound = rel.abs() * (2 * tol + tol / s.abs() + tol / e.abs()) + tol
    err = (got["relative"] - rel).abs()
    assert (err[ok] <= bound[ok]).all(), (err[ok].max().item(), (err[ok] / bound[ok]).max().item())


def test_suggestion_is_the_greedy_token(small, layout):
    """Greedy-generate a window, then score prompt + output: at every generated position where the processor chain leaves the raw
    argmax in place, `suggested` is the generated token wherever the top-2 logit gap exceeds 1e-4 (bench.py's oracle_check rule)."""
    from mapperatorinator_b200.server import model_generate, model_score
    from oracle.generate import Processors
    cfg, model = small
    g = torch.Generator().manual_seed(9)
    prompt = torch.cat([torch.tensor([[3700, 3705, 1, 9]]), torch.randint(17, 3600, (1, 60), generator=g)], dim=1)
    P, new = prompt.shape[1], 96
    gk = dict(do_sample=False, num_beams=1, max_length=P + new, min_new_tokens=new, types_first=True, temperature=0.9,
              timing_temperature=0.1, lookback_time=0.0, lookahead_time=0.0, context_type="map")
    pcm = cases.model_pcm(cfg, 1, 5)
    ids, _ = model_generate(model, layout, dict(inputs=pcm, decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0)), dict(gk))
    mk = dict(inputs=pcm, decoder_input_ids=ids, decoder_attention_mask=torch.ones_like(ids, dtype=torch.bool))
    sc = model_score(model, mk, dict(precision="fp32"))
    logits = model.forward(pcm, ids, mk["decoder_attention_mask"]).logits.cpu()
    pr = Processors(layout, 1, P, gk)
    checked = 0
    for t in range(P, ids.shape[1]):
        z = logits[0, t - 1]
        processed = pr(ids[:, :t], z[None].clone())[0]
        top = torch.topk(z, 2).values
        if int(processed.argmax()) != int(z.argmax()) or float(top[0] - top[1]) <= 1e-4:
            continue
        assert int(sc["suggested"][0, t]) == int(ids[0, t]), t
        checked += 1
    assert checked >= new // 2, checked


def test_rejections(tiny):
    from mapperatorinator_b200.server import model_score
    cfg, _, model = tiny
    ids = torch.tensor([[3700, 3705, 1, 9, 3645, 30]])
    mk = _mk(cfg, ids, ids.ne(0), 1)
    with pytest.raises(ValueError, match="guided"):
        model_score(model, dict(mk, negative_prompt=ids.clone()), dict(cfg_scale=2.0))
    with pytest.raises(ValueError, match="max_batch"):
        model.engine.score_tokens(list(range(4)) + [0], ids.repeat(5, 1), None)
    with pytest.raises(ValueError, match="tgt_seq_len"):
        model.engine.score_tokens([0], torch.full((1, cfg.tgt_seq_len + 1), 17), None)
    for bad in (cfg.vocab_size_in, -1):
        with pytest.raises(ValueError, match="token ids"):
            model_score(model, _mk(cfg, torch.tensor([[3700, bad, 1]]), None, 1), {})
    # an encoder slot outside the resident ones, or one slot per row missing, is refused before anything is launched: by the Python
    # wrapper, and by the engine itself for a caller of the C ABI
    from mapperatorinator_b200 import _lib
    eng, lib = model.engine, _lib.load()
    before = lib.mb200_launch_count()
    with pytest.raises(ValueError, match="encoder slots"):
        eng.forward_logits([eng.max_windows], ids, None)
    with pytest.raises(ValueError, match="encoder slots"):
        eng.forward_logits([0, 1], ids, None)
    B, L = ids.shape
    a = np.ascontiguousarray(ids.numpy().astype(np.int64))
    slots = np.array([eng.max_windows], dtype=np.int32)
    logits = torch.empty(B, L, cfg.vocab_size_out, device="cuda")
    assert lib.mb200_model_forward_logits(eng.handle, slots.ctypes.data, B, a.ctypes.data, None, L, 0, logits.data_ptr(), None) != 0
    assert b"encoder slot out of range" in lib.mb200_last_error()
    stats = [torch.empty(B, L, device="cuda") for _ in range(3)] + [torch.empty(B, L, device="cuda", dtype=torch.int64)]
    assert lib.mb200_model_score_tokens(eng.handle, slots.ctypes.data, B, a.ctypes.data, None, L, 0, *(t.data_ptr() for t in stats),
                                        None) != 0
    assert b"encoder slot out of range" in lib.mb200_last_error()
    assert lib.mb200_launch_count() == before


def test_generate_after_score_matches_fixture(tiny, layout):
    """A score call of the longest fixture prompt first, then a left-padded look-back generate case: the projection scratch and
    the prefill buffers the score call used must not leak into the generate call."""
    from mapperatorinator_b200.server import model_generate, model_score
    cfg, _, model = tiny
    gold = np.load(os.path.join(GOLDEN, "score_reference.npz"))
    ids, mask = torch.from_numpy(gold["ids"]), torch.from_numpy(gold["mask"])
    model_score(model, _mk(cfg, ids, mask, PCM_SEED), {})
    gen_gold = np.load(os.path.join(GOLDEN, "generate_reference.npz"))
    for name in ("b2_leftpad_lookback", "b1_eos_stop"):
        prompt, neg, gk, seed = cases.generate_cases()[name]
        mk = dict(inputs=cases.model_pcm(cfg, prompt.shape[0], seed), decoder_input_ids=prompt, decoder_attention_mask=prompt.ne(0))
        got, _ = model_generate(model, layout, mk, dict(gk))
        assert np.array_equal(got.numpy(), gen_gold[f"torchaudio/{name}/ids"]), name
