"""Song-level host logic around the engine: window segmentation, the sequential window loop with resident encoder
states, and song-sharded multi-GPU execution.

Reference behaviour being restructured (SURVEY §8f N1, F5):
  * `Preprocessor.segment` / `window` (osuT5/osuT5/inference/preprocessor.py:41-102): zero-pad to the stride grid and take
    strided windows of (src_seq_len - 1) * hop samples; sequential stride = int(samples_per_seq * (1 - lookback - lookahead)).
  * `Processor.generate_sequential` (osuT5/osuT5/inference/processor.py:308-368): one `model_generate` call per window with
    batch size 1, each call RE-RUNNING the encoder; window i+1's prompt is built from window i's tokens.
Here the encoder runs ONCE over all windows of the song (its output depends only on the audio), the cross-attention K/V of
every window stay resident in HBM, and the sequential loop only runs prefill + the token loop per window.  Results are
identical to calling `server.model_generate` per window (same kernels, same order).

Multi-GPU: songs are independent, so ranks take whole songs (sorted by length, dealt round-robin) and the only collective
is the terminal gather of the emitted token streams (`gather_token_streams`).
"""
from __future__ import annotations

from collections import deque
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .config import ModelConfig
from .token_layout import TokenLayout


def segment(samples: np.ndarray, cfg: ModelConfig, lookback: float = 0.5, lookahead: float = 0.4, parallel: bool = False
            ) -> Tuple[torch.Tensor, torch.Tensor, float]:
    """`Preprocessor.segment` (preprocessor.py:41-92) without begin/end padding options: returns (windows (n, S) f32,
    window start times in ms (n,) i32, song_length ms)."""
    S = cfg.samples_per_window
    sr = cfg.mel.sample_rate
    stride = S if parallel else int(S * (1 - lookback - lookahead))
    song_length = len(samples) / sr * 1000
    samples = np.asarray(samples, dtype=np.float32)
    pad = (stride - (len(samples) - S) % stride) % stride if len(samples) > S else S - len(samples)
    samples = np.pad(samples, [0, pad])
    n = (len(samples) - S) // stride + 1
    idx = np.arange(n)[:, None] * stride + np.arange(S)[None, :]
    windows = torch.from_numpy(samples[idx])
    times = torch.from_numpy((np.arange(n) * stride * 1000 / sr).astype(np.int32))
    return windows, times, song_length


def segment_device(samples: torch.Tensor, cfg: ModelConfig, lookback: float = 0.5, lookahead: float = 0.4, parallel: bool = False) -> torch.Tensor:
    """`segment` for a device-resident signal (the output of `audio.load_pcm`): the same padding / stride arithmetic, windows gathered on the
    device.  Returns windows (n, S) f32."""
    S = cfg.samples_per_window
    stride = S if parallel else int(S * (1 - lookback - lookahead))
    n_s = samples.shape[0]
    pad = (stride - (n_s - S) % stride) % stride if n_s > S else S - n_s
    x = torch.nn.functional.pad(samples.float(), (0, pad))
    return x.unfold(0, S, stride).contiguous()


PromptFn = Callable[[int, List[List[int]]], List[int]]


class SongDecoder:
    """Sequential decode of one song (or a batch of songs in lock-step) over resident encoder slots."""

    def __init__(self, model, layout: TokenLayout):
        self.model = model                 # B200Mapperatorinator
        self.engine = model.engine
        self.layout = layout

    def encode_song(self, windows: torch.Tensor, slot_begin: int = 0) -> None:
        """All windows of a song through mel + encoder + cross-K/V in one batched pass (device or pinned-host input)."""
        w = windows if windows.is_cuda else windows.to(self.model.device, non_blocking=True)
        self.engine.encode(w.float(), slot_begin=slot_begin)

    def decode_windows(self, n_windows: int, prompt_fn: PromptFn, generate_kwargs_fn: Callable[[int], dict], slot_begin: int = 0
                       ) -> List[List[int]]:
        """The dependency chain of generate_sequential: window i's prompt is `prompt_fn(i, generated_so_far)`."""
        streams: List[List[int]] = []
        for i in range(n_windows):
            prompt = torch.tensor([prompt_fn(i, streams)], dtype=torch.long)
            ids = self.engine.generate([slot_begin + i], prompt, prompt.ne(self.layout.pad_id), self.layout, generate_kwargs_fn(i),
                                       position_rule=self.model.position_rule)
            streams.append(ids[0, prompt.shape[1]:].tolist())
        return streams


    def decode_songs(self, n_songs: int, n_windows: int, prompt_fn: Callable[[int, int, List[List[int]]], List[int]],
                     generate_kwargs_fn: Callable[[int], dict], windows_per_song: Optional[int] = None) -> List[List[List[int]]]:
        """`n_songs` songs of equal window count decoded in LOCK-STEP (BASELINE configs[3]: 8 songs per GPU): window i of every
        song is one batch-`n_songs` `generate()` call over the resident encoder slots (song s, window i at slot
        s * windows_per_song + i).  `prompt_fn(s, i, streams_of_song_s)` must return prompts of equal length across songs.
        Returns streams[s][i]."""
        stride = windows_per_song or n_windows
        streams: List[List[List[int]]] = [[] for _ in range(n_songs)]
        for i in range(n_windows):
            prompts = [prompt_fn(s, i, streams[s]) for s in range(n_songs)]
            assert len({len(p) for p in prompts}) == 1, "lock-step batch needs equal prompt lengths (pad on the left otherwise)"
            prompt = torch.tensor(prompts, dtype=torch.long)
            ids = self.engine.generate([s * stride + i for s in range(n_songs)], prompt, prompt.ne(self.layout.pad_id), self.layout,
                                       generate_kwargs_fn(i), position_rule=self.model.position_rule)
            for s in range(n_songs):
                streams[s].append(ids[s, prompt.shape[1]:].tolist())
        return streams

    def decode_songs_ragged(self, window_counts: Sequence[int], prompt_fn: Callable[[int, int, List[List[int]]], List[int]],
                            generate_kwargs_fn: Callable[[int, int], dict], windows_per_song: Optional[int] = None
                            ) -> List[List[List[int]]]:
        """`decode_songs` for real prompts: song s has `window_counts[s]` windows (song s, window i at slot s * windows_per_song + i),
        window i of every song that still has one is one row of a ragged `generate_ragged` call, so prompts may differ in length
        (`prompt_fn(s, i, streams_of_song_s)`) and rows in kind (`generate_kwargs_fn(s, i)`: first and last windows of different songs
        share a step).  A song drops out of the batch when it ends.  Each stream equals `decode_windows` run on that song alone.
        Returns streams[s][i]."""
        stride = windows_per_song or max(window_counts)
        streams: List[List[List[int]]] = [[] for _ in window_counts]
        for i in range(max(window_counts)):
            live = [s for s, n in enumerate(window_counts) if i < n]
            prompts = [prompt_fn(s, i, streams[s]) for s in live]
            outs = self.engine.generate_ragged([(s * stride + i, torch.tensor(p, dtype=torch.long), generate_kwargs_fn(s, i), None)
                                                for s, p in zip(live, prompts)], self.layout)
            for s, p, ids in zip(live, prompts, outs):
                streams[s].append(ids[0, len(p):].tolist())
        return streams

    def decode_songs_continuous(self, window_counts: Sequence[int], prompt_fn: Callable[[int, int, List[List[int]]], List[int]],
                                generate_kwargs_fn: Callable[[int, int], dict], windows_per_song: Optional[int] = None
                                ) -> List[List[List[int]]]:
        """`decode_songs_ragged` without the per-window barrier: the songs share one decode stream, and song s's window i + 1 is
        admitted as soon as its window i has finished, whatever the other songs' windows are doing.  Same arguments and slots
        (song s, window i at slot s * windows_per_song + i); each stream equals `decode_windows` run on that song alone.
        Returns streams[s][i]."""
        stride = windows_per_song or max(window_counts, default=0)
        streams: List[List[List[int]]] = [[] for _ in window_counts]
        ready = deque(s for s, n in enumerate(window_counts) if n > 0)
        if not ready:
            return streams
        with self.engine.open_stream(self.layout, min(len(ready), self.engine.max_batch)) as stream:
            live = {}                      # row -> (song, prompt length)
            while ready or live:
                while ready and stream.free_rows:
                    s = ready.popleft()
                    i = len(streams[s])
                    p = prompt_fn(s, i, streams[s])
                    row = stream.admit(s * stride + i, torch.tensor(p, dtype=torch.long), generate_kwargs_fn(s, i))
                    live[row] = (s, len(p))
                # a song whose window is running has its next window waiting for that row
                waiting = len(ready) + sum(1 for s, _ in live.values() if len(streams[s]) + 1 < window_counts[s])
                for row, ids in stream.run(waiting=waiting):
                    s, P = live.pop(row)
                    streams[s].append(ids[0, P:].tolist())
                    if len(streams[s]) < window_counts[s]:
                        ready.append(s)
        return streams


def trim_predicted_tokens(tokens: Sequence[int], layout: TokenLayout, context_type: Optional[str] = "map", lookback_ms: float = 0.0,
                          lookahead_max_ms: float = 0.0, trim_lookback: bool = False, trim_lookahead: bool = False,
                          types_first: bool = True) -> List[int]:
    """Token-level half of `Processor.add_predicted_tokens_to_context` (processor.py:1030-1043): what a window's generated ids
    contribute to the next window's prompt.  Trailing eos / context-eos ids are dropped; if the stream then ends in a time shift
    that only stopped the generation — inside the look-ahead zone (`trim_lookahead`, ids from the time shift of `lookahead_max_ms`
    = (1 - lookahead) * window to the end of the range, processor.py:86-88) or inside the look-back zone (`trim_lookback`, ids
    below the time shift of `lookback_ms`, processor.py:84-85) — that time shift goes too, together with the type token in front
    of it when `types_first`.  (The event-level half — `_decode`, `update_event_times`, `_trim_events_after_time` — is the
    reference's control plane and stays there.)"""
    t = list(tokens)
    ends = {layout.eos_id}
    if context_type is not None and context_type in layout.context_eos:
        ends.add(layout.context_eos[context_type])
    while t and t[-1] in ends:
        t.pop()
    if t:
        lb = range(layout.time_shift_start, layout.lookback_end(lookback_ms))
        la = range(layout.lookback_end(lookahead_max_ms), layout.time_shift_end)
        if (trim_lookahead and t[-1] in la) or (trim_lookback and t[-1] in lb):
            t = t[:-2] if types_first else t[:-1]
    return t


def shard_songs(lengths: Sequence[float], world_size: int) -> List[List[int]]:
    """Songs sorted by length (longest first), dealt round-robin: rank r gets shard[r] (indices into `lengths`)."""
    order = sorted(range(len(lengths)), key=lambda i: (-lengths[i], i))
    shards: List[List[int]] = [[] for _ in range(world_size)]
    for k, i in enumerate(order):
        shards[k % world_size].append(i)
    return shards


def gather_token_streams(local_streams: List[List[int]], local_song_ids: List[int], device: Optional[torch.device] = None
                         ) -> Optional[dict]:
    """The one collective of the inference path: all ranks contribute their songs' token streams; rank 0 gets
    {song_id: tokens}.  Two all_gathers (counts, then padded int32 ids), a few MB at most — latency-bound over NVLink.
    Works with the `nccl` backend on GPUs and `gloo` on CPU (tests)."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return dict(zip(local_song_ids, local_streams))
    ws, rank = dist.get_world_size(), dist.get_rank()
    dev = device or (torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu"))
    n_local = torch.tensor([len(local_streams), max([len(s) for s in local_streams], default=0)], dtype=torch.int64, device=dev)
    meta = [torch.zeros_like(n_local) for _ in range(ws)]
    dist.all_gather(meta, n_local)
    max_songs = int(max(m[0] for m in meta)); max_len = int(max(m[1] for m in meta))
    buf = torch.full((max_songs, max_len + 2), -1, dtype=torch.int32, device=dev)      # [song_id, length, tokens...]
    for j, (sid, s) in enumerate(zip(local_song_ids, local_streams)):
        buf[j, 0] = sid; buf[j, 1] = len(s)
        if s:
            buf[j, 2:2 + len(s)] = torch.tensor(s, dtype=torch.int32, device=dev)
    out = [torch.empty_like(buf) for _ in range(ws)]
    dist.all_gather(out, buf)
    if rank != 0:
        return None
    res = {}
    for t in out:
        t = t.cpu()
        for row in t:
            if row[0] >= 0:
                res[int(row[0])] = row[2:2 + int(row[1])].tolist()
    return res
