"""The CPU oracle, request by request, against the unmodified reference's batch-1 `server.model_generate` outputs for the ragged
request sets (tests/golden/ragged_reference.npz, written by oracle/make_ragged_golden.py).  Runs anywhere: no GPU, no reference
checkout."""
import os

import numpy as np
import pytest

from mapperatorinator_b200 import tiny_model_config
from mapperatorinator_b200.weights import init_model_state_dict
from oracle import cases, generate, ragged

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REQUESTS = [(name, r) for name, reqs in ragged.ragged_cases().items() for r in range(len(reqs))]


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "ragged_reference.npz"))


@pytest.fixture(scope="module")
def tiny():
    cfg = tiny_model_config(mel=cases.MODEL_FLAVOURS["torchaudio"])
    return cfg, init_model_state_dict(cfg, 0)


@pytest.mark.parametrize("name,r", REQUESTS)
def test_request_ids_equal_reference(gold, tiny, layout, name, r):
    cfg, sd = tiny
    req = ragged.ragged_cases()[name][r]
    ids, stats = generate.model_generate(sd, cfg, layout, ragged.model_kwargs(cfg, req), dict(req["gk"]))
    assert np.array_equal(ids.numpy(), gold[f"{name}/{r}/ids"])
    assert stats["generated_tokens_per_sample"] == gold[f"{name}/{r}/counts"].tolist()


def test_fixture_covers_the_stop_and_split_cases(gold, layout):
    """What the request sets are there for: in `mixed_stops` one request ends on a natural EOS several steps before the others, one
    runs into its max_length, and a max_length <= 128 (single 128-key split) sits beside one > 128 (64-key splits)."""
    reqs = ragged.ragged_cases()["mixed_stops"]
    new, by_eos = [], []
    for r, req in enumerate(reqs):
        ids = gold[f"mixed_stops/{r}/ids"]
        gk = req["gk"]
        new.append(ids.shape[1] - req["prompt"].shape[1])
        by_eos.append(ids.shape[1] < gk["max_length"] and int(ids[0, -1]) in layout.eos_token_ids(gk["lookback_time"], gk["lookahead_time"], gk["context_type"]))
    assert any(by_eos) and min(n for n, e in zip(new, by_eos) if e) + 4 <= max(new)
    assert any(gold[f"mixed_stops/{r}/ids"].shape[1] == req["gk"]["max_length"] for r, req in enumerate(reqs))
    lengths = [req["gk"]["max_length"] for req in reqs]
    assert min(lengths) <= 128 < max(lengths)
    kinds = {(req["gk"]["lookback_time"] > 0, req["gk"]["lookahead_time"] > 0, req["gk"]["context_type"]) for req in ragged.ragged_cases()["mixed_windows"]}
    assert {(False, True, "map"), (True, True, "map"), (True, True, "kiai"), (True, False, "map")} <= kinds
