"""Oracle: raw PCM -> mel spectrogram, both front ends of `MelSpectrogram` (osuT5/osuT5/model/spectrogram.py:7-92).

TEST INFRASTRUCTURE (see oracle/__init__.py).

* `nnaudio_*`  — v29 (`configs/model/default.yaml:29-38`): nnAudio==0.3.4 `features.MelSpectrogram(sr, n_fft, n_mels,
  hop_length, center=True, fmin, fmax, pad_mode)` with its defaults `window='hann', power=2.0, htk=False, norm=1`.
  nnAudio is a third-party dependency (requirements.txt:3) that is NOT installed and NOT vendored in the original project:
  this restates its published algorithm — conv1d STFT with `cos/sin(2*pi*k*n/n_fft) * hann[n]` kernels, magnitude
  `sqrt(re^2 + im^2)`, `** power`, `mel_basis @ spec` with the librosa Slaney filterbank.  **parity unpinned** vs nnAudio.
* `torchaudio_*` — v30+ (`spectrogram.py:38-49`): restated AND pinned against the installed torchaudio through
  tests/golden/mel_reference.npz.
Output layout follows spectrogram.py:79-83: optional log1p, then permute to (B, frames, n_mels).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


# ---- filterbanks ---------------------------------------------------------------------------------------------------
def _hz_to_mel_slaney(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    with np.errstate(divide="ignore"):
        log_t = min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep
    return np.where(f >= min_log_hz, log_t, mels)


def _mel_to_hz_slaney(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), freqs)


def slaney_mel_basis(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """librosa.filters.mel(htk=False, norm=1) as vendored by nnAudio (`nnAudio/librosa_functions.py: mel`): float32
    (n_mels, 1 + n_fft//2) triangles on the Slaney scale, each scaled by 2 / (f[i+2] - f[i])."""
    n_freq = 1 + n_fft // 2
    weights = np.zeros((n_mels, n_freq), dtype=np.float32)
    fftfreqs = np.linspace(0, float(sr) / 2, n_freq, endpoint=True)
    mel_pts = np.linspace(_hz_to_mel_slaney(fmin), _hz_to_mel_slaney(fmax), n_mels + 2)
    mel_f = _mel_to_hz_slaney(mel_pts)
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    return weights


def htk_mel_basis(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """torchaudio.functional.melscale_fbanks(mel_scale='htk', norm=None), returned as (n_mels, n_freq)."""
    n_freq = 1 + n_fft // 2
    all_freqs = torch.linspace(0, sr // 2, n_freq)
    m_min = 2595.0 * math.log10(1.0 + fmin / 700.0)
    m_max = 2595.0 * math.log10(1.0 + fmax / 700.0)
    m_pts = torch.linspace(m_min, m_max, n_mels + 2)
    f_pts = 700.0 * (10 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    fb = torch.max(torch.zeros(1), torch.min(down, up))  # (n_freq, n_mels)
    return fb.T.contiguous().numpy().astype(np.float32)


def mel_basis(cfg) -> np.ndarray:
    fn = slaney_mel_basis if cfg.implementation == "nnAudio" else htk_mel_basis
    return fn(cfg.sample_rate, cfg.n_fft, cfg.n_mels, cfg.f_min, cfg.f_max)


def hann_window(n_fft: int) -> np.ndarray:
    """Periodic Hann (scipy get_window('hann', N, fftbins=True) == torch.hann_window(N)), float64."""
    n = np.arange(n_fft, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)


# ---- nnAudio flavour (v29) -----------------------------------------------------------------------------------------
def nnaudio_fourier_kernels(n_fft: int):
    """nnAudio `create_fourier_kernels(freq_scale='no')` x window, float64 -> float32 like `STFT.__init__`."""
    n_freq = n_fft // 2 + 1
    s = np.arange(n_fft, dtype=np.float64)
    k = np.arange(n_freq, dtype=np.float64)[:, None]
    w = hann_window(n_fft)[None, :]
    wsin = (np.sin(2 * np.pi * k * s / n_fft) * w).astype(np.float32)
    wcos = (np.cos(2 * np.pi * k * s / n_fft) * w).astype(np.float32)
    return torch.from_numpy(wcos)[:, None, :], torch.from_numpy(wsin)[:, None, :]


def nnaudio_melspectrogram(samples: torch.Tensor, cfg, chunk: int = 8) -> torch.Tensor:
    """(B, n) f32 -> (B, n_mels, frames) f32, nnAudio STFT(output_format='Magnitude') ** 2 then mel_basis @ spec."""
    wcos, wsin = nnaudio_fourier_kernels(cfg.n_fft)
    basis = torch.from_numpy(slaney_mel_basis(cfg.sample_rate, cfg.n_fft, cfg.n_mels, cfg.f_min, cfg.f_max))
    pad = cfg.n_fft // 2
    outs = []
    for i in range(0, samples.shape[0], chunk):
        x = samples[i:i + chunk].float()[:, None, :]
        if cfg.pad_mode == "constant":
            x = F.pad(x, (pad, pad), mode="constant", value=0.0)
        else:
            x = F.pad(x, (pad, pad), mode="reflect")
        re = F.conv1d(x, wcos, stride=cfg.hop_length)
        im = F.conv1d(x, wsin, stride=cfg.hop_length)
        spec = torch.sqrt(re.pow(2) + im.pow(2)) ** 2.0
        outs.append(torch.matmul(basis, spec))
    return torch.cat(outs, 0)


# ---- torchaudio flavour (v30+) -------------------------------------------------------------------------------------
def torchaudio_melspectrogram(samples: torch.Tensor, cfg) -> torch.Tensor:
    """torchaudio.transforms.MelSpectrogram(center=True, power=2, norm=None, mel_scale='htk') restated with
    torch.stft: (B, n) -> (B, n_mels, frames)."""
    win = torch.from_numpy(hann_window(cfg.n_fft)).float()
    st = torch.stft(samples.float(), cfg.n_fft, hop_length=cfg.hop_length, win_length=cfg.n_fft, window=win,
                    center=True, pad_mode=cfg.pad_mode, normalized=False, onesided=True, return_complex=True)
    power = st.real.pow(2) + st.imag.pow(2)                       # (B, n_freq, frames)
    fb = torch.from_numpy(htk_mel_basis(cfg.sample_rate, cfg.n_fft, cfg.n_mels, cfg.f_min, cfg.f_max))
    return torch.matmul(fb, power)


def mel_forward(samples: torch.Tensor, cfg) -> torch.Tensor:
    """`MelSpectrogram.forward` (spectrogram.py:63-83): (B, n_samples) -> (B, frames, n_mels) float32."""
    if cfg.implementation == "nnAudio":
        spec = nnaudio_melspectrogram(samples, cfg)
    else:
        spec = torchaudio_melspectrogram(samples, cfg)
    if cfg.log_scale:
        spec = torch.log1p(spec)
    return spec.permute(0, 2, 1).contiguous()
