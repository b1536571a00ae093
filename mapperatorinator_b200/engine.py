"""Python host of the engine: thin owners of the C-ABI handles.  torch is used for device memory and streams only."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .config import DiTConfig, MelConfig, ModelConfig
from .filterbank import mel_filterbank
from .token_layout import TokenLayout

VF_EOS, VF_TIMED, VF_SOS, VF_LB_EOS, VF_BEAT, VF_MANIA, VF_SCROLL = 1, 2, 4, 8, 16, 32, 64


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _mel_c(cfg: MelConfig) -> _lib.MelConfigC:
    return _lib.MelConfigC(cfg.n_fft, cfg.hop_length, cfg.n_mels, 1 if cfg.pad_mode == "reflect" else 0, 1 if cfg.log_scale else 0)


class MelEngine:
    """Stage (i).  `forward` == reference `MelSpectrogram.forward` (spectrogram.py:63-83)."""

    def __init__(self, cfg: MelConfig, mel_basis: Optional[np.ndarray] = None):
        self.cfg = cfg
        self.lib = _lib.load()
        basis = np.ascontiguousarray(mel_filterbank(cfg) if mel_basis is None else mel_basis, dtype=np.float32)
        assert basis.shape == (cfg.n_mels, cfg.n_fft // 2 + 1)
        self.handle = C.c_void_p()
        cc = _mel_c(cfg)
        _lib.check(self.lib.mb200_mel_create(C.byref(self.handle), C.byref(cc), basis.ctypes.data))

    def forward(self, samples: torch.Tensor) -> torch.Tensor:
        assert samples.is_cuda and samples.dtype == torch.float32 and samples.dim() == 2
        samples = samples.contiguous()
        B, n = samples.shape
        out = torch.empty(B, n // self.cfg.hop_length + 1, self.cfg.n_mels, device=samples.device, dtype=torch.float32)
        _lib.check(self.lib.mb200_mel_forward(self.handle, samples.data_ptr(), B, n, out.data_ptr(), _stream()))
        return out

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.mb200_mel_destroy(self.handle)
        except Exception:
            pass


def build_vflags(layout: TokenLayout, eos_ids: Sequence[int]) -> np.ndarray:
    """Per-token flag byte consumed by the fused decode step (kernels.h VF_*)."""
    f = np.zeros(layout.vocab_size_in, dtype=np.uint8)
    for ids, bit in ((eos_ids, VF_EOS), (layout.timed_token_ids(), VF_TIMED), (layout.sos_ids(), VF_SOS),
                     (layout.lookback_eos_ids(), VF_LB_EOS), (layout.beat_type_tokens(), VF_BEAT),
                     (layout.mania_type_tokens(), VF_MANIA), (layout.scroll_speed_tokens(), VF_SCROLL)):
        if len(ids):
            f[np.asarray(list(ids), dtype=np.int64)] |= bit
    return f


class _VflagsCache:
    """`build_vflags` per (layout, EOS set): sequential windows ask for the same few rows on every call.  Rows are read-only.
    A layout is keyed by identity, so it must not be changed in place once an engine has generated with it (build a new one)."""

    def __init__(self):
        self._rows: Dict[tuple, tuple] = {}

    def get(self, layout: TokenLayout, eos_ids: Sequence[int]) -> np.ndarray:
        key = (id(layout), tuple(eos_ids))
        hit = self._rows.get(key)
        if hit is None or hit[0] is not layout:       # the layout object is held, so its id cannot be reused while cached
            if len(self._rows) >= 64:
                self._rows.clear()
            f = build_vflags(layout, eos_ids)
            f.setflags(write=False)
            hit = self._rows[key] = (layout, f)
        return hit[1]


class ModelEngine:
    """Stage (ii): weights + resident encoder slots + KV arena behind `mb200_model_*`."""

    def __init__(self, cfg: ModelConfig, state_dict: Dict[str, torch.Tensor], max_windows: int = 32, max_batch: int = 16,
                 mel_basis: Optional[np.ndarray] = None, device: str = "cuda:0"):
        if not torch.cuda.is_available():
            raise RuntimeError("mapperatorinator_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.cfg = cfg
        self.device = torch.device(device)
        self.lib = _lib.load()
        self.max_windows, self.max_batch = max_windows, max_batch
        self._vflags = _VflagsCache()
        basis = np.ascontiguousarray(mel_filterbank(cfg.mel) if mel_basis is None else mel_basis, dtype=np.float32)
        cc = _lib.ModelConfigC(cfg.d_model, cfg.encoder_layers, cfg.decoder_layers, cfg.heads, cfg.ffn_dim, cfg.src_seq_len,
                               cfg.tgt_seq_len, cfg.vocab_size_in, cfg.vocab_size_out, _mel_c(cfg.mel), max_windows, max_batch)
        self.handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_create(C.byref(self.handle), C.byref(cc), basis.ctypes.data))
            for name, t in state_dict.items():
                if not isinstance(t, torch.Tensor) or not t.is_floating_point():
                    continue
                if t.dtype == torch.bfloat16:      # raw bits: the engine widens them and may serve the token loop from a bf16 store
                    a = t.detach().to("cpu").contiguous().view(torch.int16).numpy()
                    _lib.check(self.lib.mb200_model_set_weight_bf16(self.handle, name.encode(), a.ctypes.data, a.size))
                    continue
                a = t.detach().to("cpu", torch.float32).contiguous().numpy()
                _lib.check(self.lib.mb200_model_set_weight(self.handle, name.encode(), a.ctypes.data, a.size))
            _lib.check(self.lib.mb200_model_finalize(self.handle))
        nbytes = C.c_int32()
        _lib.check(self.lib.mb200_model_token_weight_bytes(self.handle, C.byref(nbytes)))
        self._token_weight_dtype = torch.bfloat16 if nbytes.value == 2 else torch.float32

    @property
    def token_weight_dtype(self) -> torch.dtype:
        """torch.bfloat16 when the engine holds a bf16 token-loop store (every decoder GEMV matrix and proj_out arrived as bf16: a model
        loaded at bf16 precision), else torch.float32.  Every token-loop driver then streams the bf16 store (megakernels, CUDA
        graph, ragged, stream, beam).  The results are the same bits either way: bf16 weights are widened exactly and summed in the
        fp32 order."""
        return self._token_weight_dtype

    # ---- encoder ---------------------------------------------------------------------------------------------------
    def encode(self, pcm: torch.Tensor, slot_begin: int = 0, return_states: bool = False) -> Optional[torch.Tensor]:
        """OsuTEncoder.forward + cross-K/V for `pcm` (n, samples_per_window) CUDA f32, into slots [slot_begin, +n)."""
        assert pcm.is_cuda and pcm.dtype == torch.float32 and pcm.dim() == 2 and pcm.shape[1] == self.cfg.samples_per_window
        pcm = pcm.contiguous()
        n = pcm.shape[0]
        out = None
        if return_states:
            out = torch.empty(n, self.cfg.max_source_positions, self.cfg.d_model, device=pcm.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_encode(self.handle, pcm.data_ptr(), n, slot_begin, out.data_ptr() if out is not None else None,
                                                   _stream()))
        return out

    # ---- decoder ---------------------------------------------------------------------------------------------------
    def _generate_params(self, layout: TokenLayout, generate_kwargs: dict, position_rule: str = "arange"):
        """generate_kwargs (server.py:83-134 names) -> the C struct + the EOS id set."""
        gk = dict(generate_kwargs)
        t = float(gk.get("temperature", 1.0))
        types_first = bool(gk.get("types_first", False))
        lookback_time = float(gk.get("lookback_time", 0.0))
        lookahead_time = float(gk.get("lookahead_time", 0.0))
        ctx = gk.get("context_type")
        eos_ids = layout.eos_token_ids(lookback_time, lookahead_time, ctx)
        p = _lib.GenerateParamsC()
        p.cfg_scale = float(gk.get("cfg_scale", 1.0))
        p.timeshift_bias = float(gk.get("timeshift_bias", 0))
        p.types_first = int(types_first)
        p.temperature = t
        p.timing_temperature = float(gk.get("timing_temperature", t))
        p.mania_column_temperature = float(gk.get("mania_column_temperature", t))
        p.taiko_hit_temperature = float(gk.get("taiko_hit_temperature", t))
        conds = []
        if types_first:  # logit_processors.py:62-71
            if p.timing_temperature != t and layout.beat_type_tokens():
                conds.append((p.timing_temperature, 1, VF_BEAT))
            if p.mania_column_temperature != t and layout.mania_type_tokens():
                conds.append((p.mania_column_temperature, 3, VF_MANIA))
            if p.taiko_hit_temperature != t and layout.scroll_speed_tokens():
                conds.append((p.taiko_hit_temperature, 1, VF_SCROLL))
        p.n_cond = len(conds)
        for i, (ct, off, fl) in enumerate(conds):
            p.cond_temp[i], p.cond_offset[i], p.cond_flag[i] = ct, off, fl
        p.lookback_on = int(lookback_time > 0)
        p.lookback_start = layout.time_shift_start
        p.lookback_end = layout.lookback_end(lookback_time) if lookback_time > 0 else layout.time_shift_start
        p.do_sample = int(bool(gk.get("do_sample", False)))
        p.top_k = int(gk.get("top_k", 0) or 0)
        p.top_p = float(gk.get("top_p", 1.0) if gk.get("top_p") is not None else 1.0)
        p.top_p_cut = 1.0 - float(gk.get("top_p", 1.0) if gk.get("top_p") is not None else 1.0)      # double arithmetic, then one rounding to f32
        p.max_length = int(gk.get("max_length", self.cfg.tgt_seq_len))
        p.min_new_tokens = int(gk.get("min_new_tokens") or 0)
        pad = gk.get("pad_token_id", layout.pad_id)
        p.pad_token_id = int(layout.pad_id if pad is None else pad)
        # The reference draws from torch's global RNG (HF _sample -> torch.multinomial), i.e. a fresh stream per call that
        # `torch.manual_seed` controls.  Same contract here: without an explicit `seed` every call takes a new 62-bit seed from
        # torch's default generator (an explicit seed pins the device RNG for tests).
        seed = gk.get("seed")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if p.do_sample else 0
        p.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        p.time_shift_start, p.time_shift_end = layout.time_shift_start, layout.time_shift_end
        p.position_rule = {"arange": 0, "mask_cumsum": 1}[position_rule]
        return p, eos_ids, gk

    def generate(self, slots: Sequence[int], prompt: torch.Tensor, prompt_mask: Optional[torch.Tensor], layout: TokenLayout,
                 generate_kwargs: dict, negative_prompt: Optional[torch.Tensor] = None,
                 negative_mask: Optional[torch.Tensor] = None, position_rule: str = "arange") -> torch.Tensor:
        """The token loop of `server.model_generate` for rows whose encoder states already sit in `slots`.
        Returns a CPU LongTensor (B, L) = prompt + generated, like the reference."""
        if int(generate_kwargs.get("num_beams", 1) or 1) != 1:
            return self.generate_beams(slots, prompt, prompt_mask, layout, generate_kwargs, negative_prompt, negative_mask,
                                       position_rule)[0]
        p, eos_ids, gk = self._generate_params(layout, generate_kwargs, position_rule)
        B, P = prompt.shape
        use_cfg = negative_prompt is not None and p.cfg_scale > 1.0
        ids, msk, neg, nmsk, vflags, slots_a = self._prompt_args(slots, prompt, prompt_mask, negative_prompt if use_cfg else None, layout,
                                                                 eos_ids)
        out = np.zeros((B, p.max_length), dtype=np.int64)
        out_len = C.c_int32(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_generate(
                self.handle, slots_a.ctypes.data, B, ids.ctypes.data, None if msk is None else msk.ctypes.data, P,
                None if neg is None else neg.ctypes.data, None if nmsk is None else nmsk.ctypes.data, vflags.ctypes.data,
                C.byref(p), out.ctypes.data, C.byref(out_len), _stream()))
        L = out_len.value
        return torch.from_numpy(out.reshape(-1)[: B * L].reshape(B, L).copy())

    def _prompt_args(self, slots: Sequence[int], prompt: torch.Tensor, prompt_mask: Optional[torch.Tensor],
                     negative_prompt: Optional[torch.Tensor], layout: TokenLayout, eos_ids: Sequence[int]):
        """The arguments of `generate` and `generate_beams` in the form of the C ABI -> (ids, mask | None, negative rows | None, their
        mask | None, vflags, slots).  `negative_prompt` is given only for a guided call."""
        B = prompt.shape[0]
        ids = np.ascontiguousarray(prompt.detach().cpu().numpy().astype(np.int64))
        msk = None if prompt_mask is None else np.ascontiguousarray(prompt_mask.detach().cpu().numpy().astype(np.uint8))
        neg = nmsk = None
        if negative_prompt is not None:
            neg_full = ids.copy()      # prepare_inputs_for_generation: ids.repeat(2); [:B, :neg_len] = negative prompt
            npn = negative_prompt.detach().cpu().numpy().astype(np.int64)
            neg_full[:, :npn.shape[1]] = npn
            neg = np.ascontiguousarray(neg_full)
            # the reference's negative_prompt_attention_mask is swallowed by HF generate()'s own parameter of that name
            # (transformers generation/utils.py:2142): the negative rows run with the conditional prompt's mask.
            nmsk = np.ascontiguousarray(msk.copy() if msk is not None else np.ones_like(ids, dtype=np.uint8))
        vflags = self._vflags.get(layout, eos_ids)
        slots_a = np.ascontiguousarray(np.asarray(list(slots), dtype=np.int32))
        assert slots_a.shape[0] == B
        return ids, msk, neg, nmsk, vflags, slots_a

    def _ragged_args(self, requests: Sequence[tuple], layout: TokenLayout):
        """Validates independent batch-1 requests `(slot, prompt ids (P_r,) without padding, generate_kwargs, negative prompt | None)` on
        the host (ValueError before anything is launched) -> (params, vflags, prompt ids back to back, offsets, negative rows | None,
        slots, guided) in the form of the C ABI's ragged and stream calls."""
        n = len(requests)
        params = (_lib.GenerateParamsC * n)()
        vflags = np.zeros((n, layout.vocab_size_in), dtype=np.uint8)
        prompts, negs, cfg_rows = [], [], []
        for r, (slot, prompt, gk, neg) in enumerate(requests):
            if int(gk.get("num_beams", 1) or 1) != 1:
                raise ValueError("a ragged call takes greedy or sampling requests; beam search (num_beams > 1) goes through generate()")
            p, eos_ids, _ = self._generate_params(layout, gk)
            ids = np.asarray(torch.as_tensor(prompt).detach().cpu().numpy(), dtype=np.int64).reshape(-1)
            if not 1 <= ids.shape[0] < p.max_length <= self.cfg.tgt_seq_len:
                raise ValueError(f"request {r}: need 1 <= prompt length ({ids.shape[0]}) < max_length ({p.max_length}) <= "
                                 f"{self.cfg.tgt_seq_len}")
            use_cfg = neg is not None and p.cfg_scale > 1.0
            cfg_rows.append(use_cfg)
            if not use_cfg:
                p.cfg_scale = 1.0          # generate() runs such a request without guidance
            neg_full = ids.copy()          # prepare_inputs_for_generation: the prompt with its first neg_len ids replaced
            if use_cfg:
                npn = np.asarray(torch.as_tensor(neg).detach().cpu().numpy(), dtype=np.int64).reshape(-1)
                neg_full[:npn.shape[0]] = npn
            params[r] = p
            vflags[r] = self._vflags.get(layout, eos_ids)
            prompts.append(ids); negs.append(neg_full)
        if any(cfg_rows) and not all(cfg_rows):
            raise ValueError("classifier-free guidance (negative prompt and cfg_scale > 1) on every request of a ragged call or on none")
        off = np.zeros(n + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(x) for x in prompts])
        flat = np.ascontiguousarray(np.concatenate(prompts))
        nflat = np.ascontiguousarray(np.concatenate(negs)) if cfg_rows[0] else None
        slots_a = np.ascontiguousarray(np.asarray([int(q[0]) for q in requests], dtype=np.int32))
        return params, vflags, flat, off, nflat, slots_a, cfg_rows[0]

    def generate_ragged(self, requests: Sequence[tuple], layout: TokenLayout) -> List[torch.Tensor]:
        """One token loop for independent requests `(slot, prompt ids (P_r,) without padding, generate_kwargs, negative prompt | None)`.
        Requests may differ in prompt length, `max_length`, `min_new_tokens`, window kind (`lookback_time`, `lookahead_time`,
        `context_type`), temperatures, `timeshift_bias`, sampling settings and `seed`, `cfg_scale`.  Returns one CPU LongTensor
        (1, L_r) per request, equal to `generate([slot], prompt[None], None, layout, generate_kwargs, negative_prompt)` of that
        request alone.  Classifier-free guidance is for every request of the call or for none; beam search has its own call."""
        n = len(requests)
        if n == 0:
            return []
        params, vflags, flat, off, nflat, slots_a, guided = self._ragged_args(requests, layout)
        rows = n * (2 if guided else 1)
        if rows > self.max_batch:
            raise ValueError(f"{n} requests{' x 2 (classifier-free guidance)' if guided else ''} = {rows} decoder rows; this engine "
                             f"was built with max_batch={self.max_batch}")
        ld = max(int(params[r].max_length) for r in range(n))
        out = np.zeros((n, ld), dtype=np.int64)
        out_len = np.zeros(n, dtype=np.int32)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_generate_ragged(
                self.handle, n, slots_a.ctypes.data, flat.ctypes.data, off.ctypes.data, None if nflat is None else nflat.ctypes.data,
                vflags.ctypes.data, C.cast(params, C.c_void_p), out.ctypes.data, ld, out_len.ctypes.data, _stream()))
        return [torch.from_numpy(out[r, :out_len[r]].copy())[None] for r in range(n)]

    def open_stream(self, layout: TokenLayout, capacity: int, guidance: bool = False, max_length: Optional[int] = None) -> "DecodeStream":
        """A decode stream over this engine: a token loop of `capacity` rows into which batch-1 requests are admitted while it runs
        (continuous batching).  Every request's ids equal its own `generate` call.  `guidance`: every request carries a negative prompt
        and cfg_scale > 1 (2 decoder rows each), or none does.  `max_length` caps the requests' max_length (default tgt_seq_len).
        While the stream is open the engine's other token-loop calls refuse; `encode` into slots no live row reads stays allowed."""
        return DecodeStream(self, layout, capacity, guidance, max_length)

    def generate_beams(self, slots: Sequence[int], prompt: torch.Tensor, prompt_mask: Optional[torch.Tensor], layout: TokenLayout,
                       generate_kwargs: dict, negative_prompt: Optional[torch.Tensor] = None,
                       negative_mask: Optional[torch.Tensor] = None, position_rule: str = "arange"):
        """`generate` with HF beam search (`num_beams` = K in [2, 4], do_sample False, default length_penalty / early_stopping).
        Returns (ids CPU LongTensor (B, L): the best finished hypothesis of each item, padded with `pad_token_id` or, when that
        is 0, the first EOS id, like the reference; scores CPU FloatTensor (B,): HF's `sequences_scores`)."""
        gk = dict(generate_kwargs)
        K = int(gk.get("num_beams", 1) or 1)
        if not 2 <= K <= 4:
            raise ValueError(f"num_beams={K}: beam search takes 2..4 beams (the candidates of one item live in one CTA's shared memory)")
        if gk.get("do_sample", False):
            raise ValueError("do_sample with num_beams > 1 (beam sampling) is not supported")
        if int(gk.get("num_return_sequences", 1) or 1) != 1:
            raise ValueError("num_return_sequences != 1 is not supported")
        if gk.get("length_penalty") not in (None, 1.0) or gk.get("early_stopping") not in (None, False):
            raise ValueError("beam search supports only the default length_penalty (1.0) and early_stopping (False)")
        p, eos_ids, gk = self._generate_params(layout, gk, position_rule)
        B, P = prompt.shape
        use_cfg = negative_prompt is not None and p.cfg_scale > 1.0
        rows = B * K * (2 if use_cfg else 1)
        if rows > self.max_batch:
            raise ValueError(f"beam search needs batch * num_beams{' * 2 (classifier-free guidance)' if use_cfg else ''} = {rows} "
                             f"decoder rows; this engine was built with max_batch={self.max_batch}")
        ids, msk, neg, nmsk, vflags, slots_a = self._prompt_args(slots, prompt, prompt_mask, negative_prompt if use_cfg else None, layout,
                                                                 eos_ids)
        fill = p.pad_token_id if p.pad_token_id else eos_ids[0]          # HF: `pad_token_id or eos_token_id[0]`
        out = np.zeros((B, p.max_length), dtype=np.int64)
        scores = np.zeros(B, dtype=np.float32)
        out_len = C.c_int32(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_generate_beams(
                self.handle, slots_a.ctypes.data, B, ids.ctypes.data, None if msk is None else msk.ctypes.data, P,
                None if neg is None else neg.ctypes.data, None if nmsk is None else nmsk.ctypes.data, vflags.ctypes.data,
                C.byref(p), K, int(fill), out.ctypes.data, C.byref(out_len), scores.ctypes.data, _stream()))
        L = out_len.value
        return torch.from_numpy(out.reshape(-1)[: B * L].reshape(B, L).copy()), torch.from_numpy(scores)

    def logits_chain(self, logits: torch.Tensor, ids: torch.Tensor, prompt_len: int, layout: TokenLayout, generate_kwargs: dict,
                     step: int = 0, has_last_scores: bool = False, use_cfg: bool = False):
        """Parity hook: one selection step of the fused logits-processor chain on given logits (rows, V) CUDA f32 and ids (B, L).
        Returns (scores (B, V) CUDA — what the selection sees, -inf = removed —, chosen (B,) CPU)."""
        p, eos_ids, gk = self._generate_params(layout, generate_kwargs)
        B, L = ids.shape
        a = np.ascontiguousarray(ids.detach().cpu().numpy().astype(np.int64))
        vflags = self._vflags.get(layout, eos_ids)
        logits = logits.contiguous().float()
        scores = torch.empty(B, self.cfg.vocab_size_out, device=logits.device, dtype=torch.float32)
        chosen = np.zeros(B, dtype=np.int64)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_logits_chain(self.handle, logits.data_ptr(), B, int(use_cfg), a.ctypes.data, L, int(prompt_len),
                                                         vflags.ctypes.data, C.byref(p), int(step), int(has_last_scores), scores.data_ptr(),
                                                         chosen.ctypes.data, _stream()))
        return scores, torch.from_numpy(chosen)

    def beam_step(self, logits: torch.Tensor, ids: torch.Tensor, run_scores: torch.Tensor, num_beams: int, prompt_len: int,
                  layout: TokenLayout, generate_kwargs: dict, step: int = 0, has_last_scores: bool = False, use_cfg: bool = False) -> dict:
        """Parity hook: one beam-search selection step on given logits (rows, V) CUDA f32, running sequences ids (B*K, L) and running
        scores (B*K,), from an empty finished store.  Returns a dict of CPU tensors: logprobs (B*K, V) processed log-probs, top (B*K)
        the first K candidates per item as flat indices beam * V + token, parent / token / score (B*K) the new running beams
        (parent = batch row), fin_score / fin_len / fin_flag (B*K) and fin_ids (B*K, L + 1) the finished store."""
        p, eos_ids, gk = self._generate_params(layout, generate_kwargs)
        BK, L = ids.shape
        B = BK // num_beams
        a = np.ascontiguousarray(ids.detach().cpu().numpy().astype(np.int64))
        rs = np.ascontiguousarray(run_scores.detach().cpu().numpy().astype(np.float32))
        vflags = self._vflags.get(layout, eos_ids)
        logits = logits.contiguous().float()
        lp = torch.empty(BK, self.cfg.vocab_size_out, device=logits.device, dtype=torch.float32)
        out = dict(top=np.zeros(BK, np.int32), parent=np.zeros(BK, np.int32), token=np.zeros(BK, np.int64), score=np.zeros(BK, np.float32),
                   fin_score=np.zeros(BK, np.float32), fin_len=np.zeros(BK, np.int32), fin_flag=np.zeros(BK, np.uint8),
                   fin_ids=np.zeros((BK, L + 1), np.int64))
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_beam_step(
                self.handle, logits.data_ptr(), B, int(num_beams), int(use_cfg), a.ctypes.data, L, int(prompt_len), vflags.ctypes.data,
                C.byref(p), rs.ctypes.data, int(step), int(has_last_scores), lp.data_ptr(), out["top"].ctypes.data,
                out["parent"].ctypes.data, out["token"].ctypes.data, out["score"].ctypes.data, out["fin_score"].ctypes.data,
                out["fin_len"].ctypes.data, out["fin_flag"].ctypes.data, out["fin_ids"].ctypes.data, _stream()))
        res = {k: torch.from_numpy(v) for k, v in out.items()}
        res["logprobs"] = lp.cpu()
        return res

    def forward_logits(self, slots: Sequence[int], ids: torch.Tensor, mask: Optional[torch.Tensor],
                       position_rule: str = "arange") -> torch.Tensor:
        a, m, slots_a = self._score_args(slots, ids, mask)
        B, L = a.shape
        out = torch.empty(B, L, self.cfg.vocab_size_out, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_forward_logits(self.handle, slots_a.ctypes.data, B, a.ctypes.data,
                                                           None if m is None else m.ctypes.data, L,
                                                           {"arange": 0, "mask_cumsum": 1}[position_rule], out.data_ptr(), _stream()))
        return out

    def _score_args(self, slots: Sequence[int], ids: torch.Tensor, mask: Optional[torch.Tensor]):
        """Validates a teacher-forced call (`forward_logits`, `score_tokens`) on the host (ValueError before anything is launched)
        -> (ids, mask, slots) as numpy arrays."""
        if ids.dim() != 2:
            raise ValueError(f"ids must be [B, L], got shape {tuple(ids.shape)}")
        B, L = ids.shape
        slots = list(slots)
        if len(slots) != B:
            raise ValueError(f"{B} rows need {B} encoder slots, got {len(slots)}")
        if not 1 <= B <= self.max_batch:
            raise ValueError(f"{B} rows; this engine was built with max_batch={self.max_batch}")
        if not 1 <= L <= self.cfg.tgt_seq_len:
            raise ValueError(f"length {L} is outside 1..tgt_seq_len={self.cfg.tgt_seq_len}")
        if any(not 0 <= s < self.max_windows for s in slots):
            raise ValueError(f"encoder slots must lie in 0..{self.max_windows - 1}")
        a = np.ascontiguousarray(ids.detach().cpu().numpy().astype(np.int64))
        if a.min() < 0 or a.max() >= self.cfg.vocab_size_in:
            raise ValueError(f"token ids must lie in 0..{self.cfg.vocab_size_in - 1}")
        if mask is not None and tuple(mask.shape) != (B, L):
            raise ValueError(f"mask shape {tuple(mask.shape)} differs from ids shape {(B, L)}")
        m = None if mask is None else np.ascontiguousarray(mask.detach().cpu().numpy().astype(np.uint8))
        return a, m, np.ascontiguousarray(np.asarray(slots, dtype=np.int32))

    def score_tokens(self, slots: Sequence[int], ids: torch.Tensor, mask: Optional[torch.Tensor],
                     position_rule: str = "arange") -> Dict[str, torch.Tensor]:
        """Per-token scores of the teacher-forced pass `forward_logits` runs on the same arguments (MaiMod, processor.py:519-525),
        without the [B, L, V] logits ever existing.  Returns device tensors [B, L] indexed by the scored token j: `entropy`,
        `surprisal`, `relative` (float32; NaN in column 0, and in surprisal / relative where ids[b, j] >= vocab_size_out) and
        `suggested` (int64 argmax of the logits row j - 1; -1 in column 0).  Every position is scored whatever the mask says."""
        a, m, slots_a = self._score_args(slots, ids, mask)
        B, L = a.shape
        out = {k: torch.empty(B, L, device=self.device, dtype=torch.float32) for k in ("entropy", "surprisal", "relative")}
        out["suggested"] = torch.empty(B, L, device=self.device, dtype=torch.int64)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_model_score_tokens(self.handle, slots_a.ctypes.data, B, a.ctypes.data,
                                                         None if m is None else m.ctypes.data, L,
                                                         {"arange": 0, "mask_cumsum": 1}[position_rule], out["entropy"].data_ptr(),
                                                         out["surprisal"].data_ptr(), out["relative"].data_ptr(),
                                                         out["suggested"].data_ptr(), _stream()))
        return out

    def set_option(self, name: str, value: int) -> None:
        _lib.check(self.lib.mb200_model_set_option(self.handle, name.encode(), int(value)))

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.mb200_model_destroy(self.handle)
        except Exception:
            pass


class DecodeStream:
    """An open decode stream of a `ModelEngine` (see `ModelEngine.open_stream`); a context manager that closes it on exit.
    `admit` puts a request into a free row, `run` advances every live row by a burst of token steps and hands back the requests
    that finished, whose rows are free again at once."""

    def __init__(self, engine: ModelEngine, layout: TokenLayout, capacity: int, guidance: bool, max_length: Optional[int]):
        self.engine, self.layout = engine, layout
        self.capacity, self.guidance = int(capacity), bool(guidance)
        self.max_length = int(engine.cfg.tgt_seq_len if max_length is None else max_length)
        rows = self.capacity * (2 if self.guidance else 1)
        if not 1 <= rows <= engine.max_batch:
            raise ValueError(f"a stream of {self.capacity} rows{' x 2 (classifier-free guidance)' if self.guidance else ''} = {rows} "
                             f"decoder rows; this engine was built with max_batch={engine.max_batch}")
        if not 2 <= self.max_length <= engine.cfg.tgt_seq_len:
            raise ValueError(f"max_length cap {self.max_length} outside 2..{engine.cfg.tgt_seq_len}")
        self._busy: Dict[int, int] = {}            # row -> prompt length, from admission until its request is handed back
        self.steps = 0                             # token steps replayed so far (the first token of a request comes with its admission)
        self.handle = C.c_void_p()
        with torch.cuda.device(engine.device):
            _lib.check(engine.lib.mb200_stream_open(engine.handle, self.capacity, int(self.guidance), self.max_length,
                                                    C.byref(self.handle), _stream()))

    @property
    def free_rows(self) -> int:
        return self.capacity - len(self._busy)

    @property
    def live_rows(self) -> int:
        return len(self._busy)

    def admit(self, slot: int, prompt, generate_kwargs: dict, negative_prompt=None) -> int:
        """Admits one batch-1 request (prompt ids (P,) without padding, its encoder states already in `slot`) into a free row and
        queues its prefill and first token; returns the row.  Validation and parameters are those of `generate_ragged`."""
        if not self.handle:
            raise RuntimeError("the stream is closed")
        params, vflags, flat, off, nflat, slots_a, guided = self.engine._ragged_args([(slot, prompt, generate_kwargs, negative_prompt)],
                                                                                     self.layout)
        if guided != self.guidance:
            raise ValueError(f"a {'guided' if guided else 'unguided'} request (negative prompt and cfg_scale > 1) does not fit a "
                             f"{'guided' if self.guidance else 'unguided'} stream")
        if params[0].max_length > self.max_length:
            raise ValueError(f"max_length {params[0].max_length} exceeds the stream's cap of {self.max_length}")
        if not self.free_rows:
            raise ValueError(f"all {self.capacity} rows of the stream are busy")
        row = np.zeros(1, dtype=np.int32)
        with torch.cuda.device(self.engine.device):
            _lib.check(self.engine.lib.mb200_stream_admit(
                self.handle, 1, slots_a.ctypes.data, flat.ctypes.data, off.ctypes.data, None if nflat is None else nflat.ctypes.data,
                vflags.ctypes.data, C.cast(params, C.c_void_p), row.ctypes.data, _stream()))
        self._busy[int(row[0])] = int(off[1])
        return int(row[0])

    def run(self, waiting: int = 0) -> List[tuple]:
        """One burst of token steps over the live rows -> [(row, ids CPU LongTensor (1, L))] for the requests that finished in it
        (prompt + generated, as `generate` returns them); their rows are free again.  `waiting`: how many requests the caller holds
        ready to admit — while any wait, bursts are short so that a freed row is refilled within a step or two."""
        if not self.handle:
            raise RuntimeError("the stream is closed")
        done_rows = np.zeros(self.capacity, dtype=np.int32)
        done_len = np.zeros(self.capacity, dtype=np.int32)
        n_done, steps = C.c_int32(0), C.c_int32(0)
        lib = self.engine.lib
        out = []
        with torch.cuda.device(self.engine.device):
            _lib.check(lib.mb200_stream_run(self.handle, int(waiting), done_rows.ctypes.data, done_len.ctypes.data, C.byref(n_done),
                                            C.byref(steps), _stream()))
            self.steps += steps.value
            for k in range(n_done.value):
                row, L = int(done_rows[k]), int(done_len[k])
                ids = np.zeros(L, dtype=np.int64)
                _lib.check(lib.mb200_stream_take(self.handle, row, ids.ctypes.data, L, _stream()))
                del self._busy[row]
                out.append((row, torch.from_numpy(ids)[None]))
        return out

    def close(self) -> None:
        if getattr(self, "handle", None):
            self.engine.lib.mb200_stream_close(self.handle)
            self.handle = C.c_void_p()
            self._busy.clear()

    def __enter__(self) -> "DecodeStream":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DiTEngine:
    """Stage (iii) behind `mb200_dit_*`."""

    def __init__(self, cfg: DiTConfig, state_dict: Dict[str, torch.Tensor], max_seq_len: int = 1024, max_batch: int = 2,
                 device: str = "cuda:0"):
        if not torch.cuda.is_available():
            raise RuntimeError("mapperatorinator_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.cfg = cfg
        self.device = torch.device(device)
        self.lib = _lib.load()
        cc = _lib.DitConfigC(cfg.hidden, cfg.depth, cfg.heads, cfg.mlp_ratio, cfg.in_channels, cfg.context_size, cfg.class_size,
                             cfg.pos_freq_dim, cfg.t_freq_dim, max_seq_len, max_batch)
        self.handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_dit_create(C.byref(self.handle), C.byref(cc)))
            for name, t in state_dict.items():
                a = t.detach().to("cpu", torch.float32).contiguous().numpy()
                _lib.check(self.lib.mb200_dit_set_weight(self.handle, name.encode(), a.ctypes.data, a.size))
            _lib.check(self.lib.mb200_dit_finalize(self.handle))
        self._mask_keep = None

    def _mask(self, mask_mode: str, band: int, dense: Optional[torch.Tensor]) -> _lib.DitMaskC:
        mm = {"none": 0, "band": 2, "dense": 3}[mask_mode]
        self._mask_keep = dense
        return _lib.DitMaskC(mm, int(band), None if dense is None else dense.data_ptr())

    def forward_with_cfg(self, x, t, c, y, cfg_scale: float, mask_mode: str = "none", band: int = 0, dense=None) -> torch.Tensor:
        N, _, T = x.shape
        x, c, y = x.contiguous().float(), c.contiguous().float(), y.contiguous().float()
        tt = np.ascontiguousarray(t.detach().cpu().numpy().astype(np.int32))
        out = torch.empty(N, self.cfg.out_channels, T, device=x.device, dtype=torch.float32)
        mk = self._mask(mask_mode, band, dense)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_dit_forward_with_cfg(self.handle, x.data_ptr(), tt.ctypes.data, c.data_ptr(), y.data_ptr(), N, T,
                                                           float(cfg_scale), C.byref(mk), out.data_ptr(), _stream()))
        return out

    def sample_loop(self, z, c, y, cfg_scale: float, schedule_rows: np.ndarray, noise: torch.Tensor,
                    inpaint: Optional[torch.Tensor] = None, mask_mode: str = "none", band: int = 0, dense=None) -> torch.Tensor:
        """schedule_rows (steps, 8) in LOOP order (first row = highest timestep); noise (steps, N, 2, T)."""
        N, _, T = z.shape
        z, c, y, noise = z.contiguous().float(), c.contiguous().float(), y.contiguous().float(), noise.contiguous().float()
        sched = np.ascontiguousarray(schedule_rows, dtype=np.float32)
        steps = sched.shape[0]
        assert noise.shape == (steps, N, 2, T)
        ip = None if inpaint is None else inpaint.to(torch.uint8).contiguous()
        out = torch.empty_like(z)
        mk = self._mask(mask_mode, band, dense)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_dit_sample_loop(self.handle, z.data_ptr(), c.data_ptr(), y.data_ptr(),
                                                      None if ip is None else ip.data_ptr(), N, T, float(cfg_scale), C.byref(mk),
                                                      sched.ctypes.data, steps, noise.data_ptr(), out.data_ptr(), _stream()))
        return out

    CURVE_TYPES = {"Bezier": 0, "PerfectCurve": 1, "Catmull": 2, "Linear": 3, None: 0}

    def set_sliders(self, sliders) -> int:
        """Register the sliders of the chunk about to be sampled: iterable of (curve_type, control-point indices, end index, length)
        with CHUNK-RELATIVE indices (empty / None clears).  Returns how many were registered."""
        sl = list(sliders or [])
        if not sl:
            _lib.check(self.lib.mb200_dit_set_sliders(self.handle, 0, None, None, None, None, None))
            return 0
        off = np.zeros(len(sl) + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(s[1]) for s in sl])
        idx = np.ascontiguousarray(np.concatenate([np.asarray(s[1], dtype=np.int32) for s in sl]))
        end = np.ascontiguousarray([int(s[2]) for s in sl], dtype=np.int32)
        typ = np.ascontiguousarray([self.CURVE_TYPES.get(s[0], 0) for s in sl], dtype=np.int32)      # anything unknown flattens as a bezier (slider_path.py:114-115)
        length = np.ascontiguousarray([float(s[3]) for s in sl], dtype=np.float32)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_dit_set_sliders(self.handle, len(sl), off.ctypes.data, idx.ctypes.data, end.ctypes.data, typ.ctypes.data,
                                                      length.ctypes.data))
        return len(sl)

    def apply_sliders(self, x: torch.Tensor) -> torch.Tensor:
        """The slider half of the `denoised_fn` closure on x (N, 2, T) CUDA f32 (returns a new tensor)."""
        x = x.contiguous().float().clone()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mb200_dit_apply_sliders(self.handle, x.data_ptr(), x.shape[0], x.shape[2], _stream()))
        return x

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.mb200_dit_destroy(self.handle)
        except Exception:
            pass
