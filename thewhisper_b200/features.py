"""Host-side constants of the log-mel front end (init-time only; the arithmetic runs in csrc/logmel.cu).

slaney mel filter bank, restated from the published algorithm that transformers implements in
TF/audio_utils.py:263-375,453-544 (mel_scale="slaney", norm="slaney"), which WhisperFeatureExtractor builds at
TF/models/whisper/feature_extraction_whisper.py:94-103 with num_frequency_bins=201, min 0 Hz, max 8 kHz.
"""
from __future__ import annotations

import numpy as np

SAMPLE_RATE = 16000
N_FFT = 400
HOP = 160


def _hz_to_mel_slaney(f: np.ndarray) -> np.ndarray:
    f = np.asarray(f, dtype=np.float64)
    min_log_hertz, min_log_mel, logstep = 1000.0, 15.0, 27.0 / np.log(6.4)
    mels = 3.0 * f / 200.0
    log_region = f >= min_log_hertz
    mels = np.where(log_region, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hertz) * logstep, mels)
    return mels


def _mel_to_hz_slaney(m: np.ndarray) -> np.ndarray:
    m = np.asarray(m, dtype=np.float64)
    min_log_hertz, min_log_mel, logstep = 1000.0, 15.0, np.log(6.4) / 27.0
    f = 200.0 * m / 3.0
    log_region = m >= min_log_mel
    return np.where(log_region, min_log_hertz * np.exp(logstep * (m - min_log_mel)), f)


def mel_filter_bank(n_mels: int = 128, n_bins: int = 1 + N_FFT // 2, sr: int = SAMPLE_RATE,
                    fmin: float = 0.0, fmax: float = 8000.0) -> np.ndarray:
    """[n_bins, n_mels] float32 triangular filters, slaney-normalised (area 2/(f_hi - f_lo))."""
    mel_lo, mel_hi = _hz_to_mel_slaney(np.array(fmin)), _hz_to_mel_slaney(np.array(fmax))
    mel_pts = np.linspace(mel_lo, mel_hi, n_mels + 2)
    filt_hz = _mel_to_hz_slaney(mel_pts)
    fft_hz = np.linspace(0, sr // 2, n_bins)
    fdiff = np.diff(filt_hz)
    slopes = filt_hz[None, :] - fft_hz[:, None]
    down = -slopes[:, :-2] / fdiff[:-1]
    up = slopes[:, 2:] / fdiff[1:]
    bank = np.maximum(0.0, np.minimum(down, up))
    enorm = 2.0 / (filt_hz[2:n_mels + 2] - filt_hz[:n_mels])
    bank = bank * enorm[None, :]
    return bank.astype(np.float32)


def pad_or_trim(audio: np.ndarray, n_samples: int) -> np.ndarray:
    """Zero-pad / truncate to the chunk length (feature_extraction_whisper.py:296-303)."""
    audio = np.asarray(audio, dtype=np.float32).reshape(-1)
    if audio.shape[0] >= n_samples:
        return audio[:n_samples]
    out = np.zeros(n_samples, dtype=np.float32)
    out[: audio.shape[0]] = audio
    return out


def num_valid_frames(n_audio_samples: int, n_samples: int) -> int:
    """Valid mel frames of a (possibly shorter) input = attention_mask[:, ::hop].sum() (feature_extraction :328-337)."""
    n = min(n_audio_samples, n_samples)
    return (n + HOP - 1) // HOP if n % HOP else n // HOP


def long_form_frames(n_audio_samples: int, n_padded: int) -> int:
    """Frames of one item in a long-form group zero-padded to n_padded samples = its row of the feature extractor's rescaled
    attention mask summed (feature_extraction_whisper.py:328-337: attention_mask[:, ::hop], minus the last column when n_padded is
    not a multiple of hop): the frames j < n_padded // hop with j * hop < n_audio_samples."""
    return min((n_audio_samples + HOP - 1) // HOP, n_padded // HOP)
