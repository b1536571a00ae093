"""mapperatorinator_b200 — H100-native (Hopper, sm_90a) engine for the Mapperatorinator inference hot path.

file PCM (e.g. 44.1 kHz 16-bit stereo) -> audio ingest (`audio.load_pcm`: the reference's resample / mono / normalise arithmetic) ->
raw 16 kHz PCM -> fused STFT+mel -> Whisper-small encoder -> KV-cached event-token decode (logits-processor chain
fused on device) -> DiT position refinement loop, behind the reference's own Python boundary
(`server.model_generate`, `Mapperatorinator`, `DiT.forward_with_cfg`, `SpacedDiffusion.p_sample_loop`).

All compute lives in `csrc/` (hand-written sm_90a CUDA behind a C ABI, see include/mapperatorinator_b200.h).
There is no CPU fallback: importing the compute entry points without the built library raises.
"""
from .config import (DiTConfig, MelConfig, ModelConfig, dit_b_config, tiny_dit_config, tiny_model_config,
                     v29_model_config)
from .token_layout import TokenLayout

__all__ = ["DiTConfig", "MelConfig", "ModelConfig", "TokenLayout", "dit_b_config", "tiny_dit_config",
           "tiny_model_config", "v29_model_config"]
