"""`Mapperatorinator`-shaped façade over the engine (the surface `model_generate` / `Processor` touch, SURVEY §8b B1).

Reference: osuT5/osuT5/model/modeling_mapperatorinator.py:60-443.  The façade owns a `ModelEngine`; `generate` follows the
HF call the reference makes (server.py:143-150) — encoder once, prefill, token loop with the logits-processor chain — but
the processors are fused on device, so instead of a `LogitsProcessorList` it receives the reference's `generate_kwargs`.
"""
from __future__ import annotations

import types
from typing import Dict, Optional

import torch

from .config import ModelConfig
from .engine import ModelEngine
from .token_layout import TokenLayout


class B200Mapperatorinator:
    main_input_name = "frames"

    def __init__(self, cfg: ModelConfig, state_dict: Dict[str, torch.Tensor], max_windows: int = 32, max_batch: int = 16,
                 device: str = "cuda:0", position_rule: str = "arange", mel_basis=None):
        self.cfg = cfg
        self.engine = ModelEngine(cfg, state_dict, max_windows=max_windows, max_batch=max_batch, device=device, mel_basis=mel_basis)
        self.device = torch.device(device)
        self.dtype = torch.float32
        self.position_rule = position_rule
        # what cache_utils.get_cache / callers read from `model.config` (cache_utils.py:27-33)
        self.config = types.SimpleNamespace(max_target_positions=cfg.max_target_positions, max_source_positions=cfg.max_source_positions,
                                            vocab_size=cfg.vocab_size_out, vocab_size_in=cfg.vocab_size_in, hidden_size=cfg.d_model)
        self.generation_config = types.SimpleNamespace(disable_compile=True)

    @classmethod
    def from_reference(cls, ref_model, **kw) -> "B200Mapperatorinator":
        """Build from a loaded reference `Mapperatorinator` (v29-style: stock Whisper backbone, no cond embedders)."""
        c = ref_model.config
        from .config import MelConfig
        b = c.backbone_config if not isinstance(c.backbone_config, dict) else types.SimpleNamespace(**c.backbone_config)
        mel = MelConfig(c.spectrogram_implementation, c.spectrogram_log_scale, c.sample_rate, c.n_fft, c.n_mels, c.hop_length,
                        c.f_min, c.f_max, c.pad_mode)
        cfg = ModelConfig(d_model=b.d_model, encoder_layers=b.encoder_layers, decoder_layers=b.decoder_layers,
                          heads=b.decoder_attention_heads, ffn_dim=b.decoder_ffn_dim, src_seq_len=c.src_seq_len,
                          tgt_seq_len=c.tgt_seq_len, vocab_size_out=c.vocab_size_out, vocab_size_in=c.vocab_size_in, mel=mel)
        for flag in ("do_style_embed", "do_difficulty_embed", "do_mapper_embed", "do_song_position_embed"):
            if getattr(c, flag, False):
                raise NotImplementedError(f"{flag}: conditioning embedders are v30+ (SURVEY §8a a3: absent at v29)")
        sd = ref_model.state_dict()
        basis = None
        for k in ("spectrogram.transform.mel_basis",):
            if k in sd:
                basis = sd[k].float().cpu().numpy()
        if "spectrogram.transform.mel_scale.fb" in sd:
            basis = sd["spectrogram.transform.mel_scale.fb"].float().cpu().numpy().T.copy()
        return cls(cfg, sd, mel_basis=basis, **kw)

    # nn.Module-ish no-ops the loaders call (model_utils.py:408-409)
    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def get_encoder(self):
        return lambda frames, **kw: (self.engine.encode(frames.to(self.device, torch.float32), 0, return_states=True),)

    def generate(self, inputs: torch.Tensor, decoder_input_ids: torch.Tensor, decoder_attention_mask: Optional[torch.Tensor] = None,
                 negative_prompt: Optional[torch.Tensor] = None, negative_prompt_attention_mask: Optional[torch.Tensor] = None,
                 tokenizer=None, generate_kwargs: Optional[dict] = None, **hf_kwargs) -> torch.Tensor:
        """Encoder + prefill + token loop for one batch of windows (re-encodes per call, as the reference does)."""
        assert tokenizer is not None, "pass the tokenizer (or a TokenLayout): the logits-processor chain is fused on device"
        layout = TokenLayout.from_tokenizer(tokenizer)
        gk = dict(generate_kwargs or {})
        gk.update(hf_kwargs)
        B = inputs.shape[0]
        self.engine.encode(inputs.to(self.device, torch.float32), slot_begin=0)
        return self.engine.generate(list(range(B)), decoder_input_ids, decoder_attention_mask, layout, gk,
                                    negative_prompt=negative_prompt, negative_mask=negative_prompt_attention_mask,
                                    position_rule=self.position_rule)

    def forward(self, frames: torch.Tensor, decoder_input_ids: torch.Tensor, decoder_attention_mask: Optional[torch.Tensor] = None,
                **kw):
        """Teacher-forced logits (`Mapperatorinator.forward`, :139-228, without the loss)."""
        B = frames.shape[0]
        self.engine.encode(frames.to(self.device, torch.float32), slot_begin=0)
        logits = self.engine.forward_logits(list(range(B)), decoder_input_ids, decoder_attention_mask, self.position_rule)
        return types.SimpleNamespace(logits=logits, loss=None)

    def score(self, frames: torch.Tensor, decoder_input_ids: torch.Tensor, decoder_attention_mask: Optional[torch.Tensor] = None
              ) -> Dict[str, torch.Tensor]:
        """Per-token entropy / surprisal / relative surprisal / suggested token of the teacher-forced pass `forward` runs
        (see `ModelEngine.score_tokens`); encodes the frames per call, as `forward` does."""
        B = frames.shape[0]
        if decoder_input_ids.shape[0] != B:
            raise ValueError(f"{decoder_input_ids.shape[0]} decoder rows for {B} windows of frames")
        if B > self.engine.max_windows:
            raise ValueError(f"{B} windows; this engine was built with max_windows={self.engine.max_windows}")
        self.engine._score_args(list(range(B)), decoder_input_ids, decoder_attention_mask)   # reject before the encoder runs
        self.engine.encode(frames.to(self.device, torch.float32), slot_begin=0)
        return self.engine.score_tokens(list(range(B)), decoder_input_ids, decoder_attention_mask, self.position_rule)

    __call__ = forward
