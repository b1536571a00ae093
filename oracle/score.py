"""Oracle of MaiMod's per-token scoring (`Processor.ai_mod`, osuT5/osuT5/inference/processor.py:519-525), restated on the
teacher-forced logits of a call and laid out as `server.model_score` returns it: [B, L] arrays indexed by the scored token j.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Plain CPU torch fp32.
"""
from __future__ import annotations

import math

import torch


def score_case(cfg):
    """B = 3 windows with about 40, 300 and 700 real tokens, left-padded to 700; ids drawn as in `cases.teacher_forcing_case`
    (uniform over the input vocabulary from id 17), so targets >= vocab_size_out occur."""
    g = torch.Generator().manual_seed(5)
    L, real = 700, (40, 300, 700)
    ids = torch.randint(17, cfg.vocab_size_in, (len(real), L), generator=g)
    for b, n in enumerate(real):
        ids[b, :L - n] = 0
    return ids, ids.ne(0)


def score_from_logits(logits: torch.Tensor, ids: torch.Tensor) -> dict:
    """logits [B, L, V] of a teacher-forced call on ids [B, L] -> entropy / surprisal / relative / suggested [B, L], plus the
    top-2 logit gap of the row each position is scored from.  Column 0 has no logits row: NaN (suggested -1).  A target
    >= V has NaN surprisal and relative (the reference would raise an IndexError there; ai_mod never scores such a token)."""
    B, L, V = logits.shape
    z = logits[:, :-1].float()
    probs = z.softmax(dim=-1)                                                           # processor.py:519
    entropy = -torch.sum(probs * torch.log2(probs + 1e-10), dim=-1)                     # :520
    y = ids[:, 1:]
    valid = y < V
    p_y = probs.gather(-1, y.clamp(max=V - 1)[..., None])[..., 0]
    surprisal = torch.where(valid, -torch.log2(p_y + 1e-10), torch.full_like(p_y, math.nan))       # :521
    relative = torch.where(entropy > 0, surprisal / entropy, torch.zeros_like(entropy))           # :522
    relative = torch.where(valid, relative, torch.full_like(relative, math.nan))
    suggested = z.argmax(dim=-1)                                                        # :525
    top2 = z.topk(2, dim=-1).values
    gap = top2[..., 0] - top2[..., 1]

    def col0(x, fill):
        return torch.cat([torch.full((B, 1), fill, dtype=x.dtype, device=x.device), x], dim=1)

    return dict(entropy=col0(entropy, math.nan), surprisal=col0(surprisal, math.nan), relative=col0(relative, math.nan),
                suggested=col0(suggested, -1), top2_gap=col0(gap, math.nan))
