"""TacotronSTFT — the mel front-end of the Tango checkpoint — on the sm_90a kernels (SURVEY.md section 8(f).2).

Drop-in for /root/reference/audioldm/audio/stft.py:136-186 as Tango builds and loads it (tango.py:19,23,27:
`TacotronSTFT(**stft_config).to(device)`, `load_state_dict(pytorch_model_stft.bin)`, `.eval()`) and as the callers of
`tango.stft` use it (inference.py:81, inference_hf.py:77 hand it to tools/torch_tools.py:57-77 `wav_to_fbank`):
`mel_spectrogram(y) -> (log-mel (B, n_mel, frames), log-magnitudes (B, bins, frames), energy (B, frames))`.

How it runs: the waveform is reflect-padded and split into bf16 hi / lo planes (tng_stft_frames); STFT.transform's strided
conv1d with the windowed Fourier basis is ONE tng_conv_gemm whose A operand is an *overlapping* strided TMA view of those
planes (row f = samples [f hop, f hop + filter_length): no im2col buffer); magnitude, log and frame energy are one pass
(tng_stft_magnitude); the mel filter bank is a second tng_conv_gemm followed by tng_log_clamp. Both contractions always
use the 3-term hi/lo split (~fp32 accuracy): a log-mel needs it and the cost is nil next to the decoder.

State: `stft_fn.forward_basis` ([2 bins, 1, filter_length]), `stft_fn.inverse_basis` (accepted, unused at inference) and
`mel_basis` ([n_mel, bins]) as in the checkpoint. Constructed without a checkpoint, the Fourier basis is rebuilt from
its definition (stft.py:26-47) and the mel filter bank from the published Slaney formula that `librosa.filters.mel`
implements (librosa is not in this image, so that default is not pinned against it; a loaded `mel_basis` replaces it).
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import lib as L
from .blocks import Buffers
from .ops import PackedConv, ceil_div

FLOOR = 1e-5   # dynamic_range_compression clip_val (audio_processing.py:85-91)


def fourier_basis(filter_length: int, win_length: int) -> torch.Tensor:
    """[2 (filter_length/2 + 1), 1, filter_length]: real then imaginary DFT rows times the periodic Hann window
    centred in the frame (stft.py:26-47)."""
    fb = np.fft.fft(np.eye(filter_length))
    cutoff = filter_length // 2 + 1
    fb = np.vstack([np.real(fb[:cutoff, :]), np.imag(fb[:cutoff, :])])
    n = np.arange(win_length)
    window = 0.5 - 0.5 * np.cos(2.0 * math.pi * n / win_length)
    lpad = (filter_length - win_length) // 2
    window = np.pad(window, (lpad, filter_length - win_length - lpad))
    return torch.FloatTensor(fb[:, None, :]) * torch.from_numpy(window).float()


def slaney_mel_basis(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: Optional[float]) -> torch.Tensor:
    """Slaney-style mel filter bank (linear below 1 kHz, log above; area-normalised triangles): the algorithm of
    `librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)` with its defaults (htk=False, norm="slaney")."""
    fmax = sr / 2.0 if fmax is None else float(fmax)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0

    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-12) / min_log_hz) / logstep, f / f_sp)

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return torch.from_numpy(w).float()


class TacotronSTFT:
    def __init__(self, filter_length, hop_length, win_length, n_mel_channels, sampling_rate, mel_fmin, mel_fmax):
        if hop_length % 8:
            raise NotImplementedError("hop_length must be a multiple of 8 samples (16-byte TMA stride)")
        if filter_length % 64:
            raise NotImplementedError("filter_length must be a multiple of 64")
        self.n_mel_channels, self.sampling_rate = n_mel_channels, sampling_rate
        self.filter_length, self.hop_length, self.win_length = filter_length, hop_length, win_length
        self.bins = filter_length // 2 + 1
        self.stft_fn = SimpleNamespace(filter_length=filter_length, hop_length=hop_length, win_length=win_length,
                                       forward_basis=fourier_basis(filter_length, win_length), inverse_basis=None)
        self.mel_basis = slaney_mel_basis(sampling_rate, filter_length, n_mel_channels, mel_fmin, mel_fmax)
        self.mel_basis_source = "slaney formula (not pinned against librosa)"
        self._device = torch.device("cpu")
        self._packed = False
        self._bufs: Optional[Buffers] = None

    # ------------------------------------------------------------------------------------------ module plumbing
    def to(self, device=None, *_a, **_k):
        if device is not None and not isinstance(device, torch.dtype):
            device = torch.device(device)
            if device != self._device:
                self._device, self._packed = device, False
        return self

    def eval(self):
        return self

    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {"stft_fn.forward_basis": self.stft_fn.forward_basis, "mel_basis": self.mel_basis}
        if self.stft_fn.inverse_basis is not None:
            sd["stft_fn.inverse_basis"] = self.stft_fn.inverse_basis
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        want = {"stft_fn.forward_basis": (2 * self.bins, 1, self.filter_length),
                "stft_fn.inverse_basis": (2 * self.bins, 1, self.filter_length),
                "mel_basis": (self.n_mel_channels, self.bins)}
        missing = [k for k in want if k not in sd]
        unexpected = [k for k in sd if k not in want]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for TacotronSTFT: missing {missing}, unexpected {unexpected}")
        for k, shp in want.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise RuntimeError(f"size mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(shp)}")
        if "stft_fn.forward_basis" in sd:
            self.stft_fn.forward_basis = sd["stft_fn.forward_basis"].detach().float().cpu()
        if "stft_fn.inverse_basis" in sd:
            self.stft_fn.inverse_basis = sd["stft_fn.inverse_basis"].detach().float().cpu()
        if "mel_basis" in sd:
            self.mel_basis = sd["mel_basis"].detach().float().cpu()
            self.mel_basis_source = "checkpoint"
        self._packed = False
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ------------------------------------------------------------------------------------------ packing
    def _pack(self):
        if self._packed:
            return
        L.require_cuda_device(self._device)
        L.load()
        dev = self._device
        nb = 2 * self.bins
        self.n_pad = ceil_div(nb, 4) * 4                         # GEMM columns: a multiple of 4 (16-byte fp32 stores)
        basis = torch.zeros(self.n_pad, self.filter_length)
        basis[:nb] = self.stft_fn.forward_basis.reshape(nb, self.filter_length)
        self._basis = PackedConv(basis, None, split=True, device=dev)
        self.c_pad = ceil_div(self.bins, 8) * 8                  # operand channels: a multiple of 8 (TMA)
        mel = torch.zeros(self.n_mel_channels, self.c_pad)
        mel[:, :self.bins] = self.mel_basis
        self._mel = PackedConv(mel, None, split=True, device=dev)
        self._bufs = Buffers(dev)
        self._packed = True

    # ------------------------------------------------------------------------------------------ forward
    def mel_rows(self, y: torch.Tensor):
        """y fp32 [B, T] on the device -> (mel fp32 [B*frames, n_mel] (log), log_mag fp32 [B*frames, bins],
        energy fp32 [B*frames], frames), rows = (batch, frame)."""
        self._pack()
        L.require_cuda(y)
        y = y.to(torch.float32).contiguous()
        B, T = y.shape
        FL, hop, pad = self.filter_length, self.hop_length, self.filter_length // 2
        if T <= pad:
            raise L.TangoB200Error(f"waveform of {T} samples is too short for reflect padding by {pad}")
        frames = 1 + T // hop                                    # conv1d output length over T + filter_length samples
        ld = ceil_div(T + 2 * pad, 8) * 8
        hi = self._bufs.get("hi", (B, ld), torch.bfloat16)
        lo = self._bufs.get("lo", (B, ld), torch.bfloat16)
        L.stft_frames(y, pad, hi, lo)
        rows = B * frames
        # STFT.transform (stft.py:52-83): every frame is a window of the padded signal, so the A operand of the basis
        # GEMM is the overlapping view (channel = sample inside the frame, w = frame index with stride hop)
        views = [L.View(t, FL, frames, 1, B, hop, ld, ld) for t in (hi, lo)]
        nkb, kh = FL // 64, self._basis.k_half
        groups = [(0, 0, 0, 0, 0, nkb), (1, 0, 0, 0, 0, nkb), (0, 0, 0, 0, kh, nkb)]   # hi*w_hi + lo*w_hi + hi*w_lo
        Fq = self._bufs.get("F", (rows, self.n_pad), torch.float32)
        L.conv_gemm(views, groups, self._basis.weight, frames, 1, B, out_f32=Fq, algo_k=FL)
        mag = self._bufs.get("mag", (rows, 2 * self.c_pad), torch.bfloat16)    # [hi | lo], pad columns stay zero
        log_mag = self._bufs.get("log_mag", (rows, self.bins), torch.float32)
        energy = self._bufs.get("energy", (rows,), torch.float32)
        L.stft_magnitude(Fq, self.bins, mag, self.c_pad, log_mag, energy, FLOOR)
        from .ops import run_linear
        mel_lin = self._bufs.get("mel_lin", (rows, self.n_mel_channels), torch.float32)
        run_linear(self._mel, mag, out_f32=mel_lin)
        mel = self._bufs.get("mel", (rows, self.n_mel_channels), torch.float32)
        L.log_clamp(mel_lin, mel, FLOOR)
        return mel, log_mag, energy, frames

    def mel_spectrogram(self, y: torch.Tensor, normalize_fun=torch.log):
        """stft.py:161-186: y (B, T) in [-1, 1] -> (mel (B, n_mel, frames), log-magnitudes (B, bins, frames),
        energy (B, frames)); like the reference it refuses input outside [-1, 1]."""
        if normalize_fun is not torch.log:
            raise NotImplementedError("only the reference default normalize_fun=torch.log is on the kernels")
        L.require_cuda_device(self._device)
        y = y.to(self._device)
        assert float(y.min()) >= -1, float(y.min())
        assert float(y.max()) <= 1, float(y.max())
        mel, log_mag, energy, frames = self.mel_rows(y)
        B = y.shape[0]
        return (mel.view(B, frames, -1).transpose(1, 2).contiguous(),
                log_mag.view(B, frames, -1).transpose(1, 2).contiguous(), energy.view(B, frames).clone())


# ---------------------------------------------------------------------------------------------- tools/torch_tools.py
def normalize_wav(waveform: torch.Tensor) -> torch.Tensor:
    """torch_tools.py:9-12."""
    waveform = waveform - torch.mean(waveform)
    return waveform / (torch.max(torch.abs(waveform)) + 1e-8) * 0.5


def pad_wav(waveform: torch.Tensor, segment_length: int) -> torch.Tensor:
    """torch_tools.py:15-24."""
    n = waveform.numel()
    if segment_length is None or n == segment_length:
        return waveform
    if n > segment_length:
        return waveform[:segment_length]
    return torch.cat([waveform, torch.zeros(segment_length - n, device=waveform.device)])


def _pad_spec(fbank: torch.Tensor, target_length: int = 1024) -> torch.Tensor:
    """torch_tools.py:27-41."""
    B, n, ch = fbank.shape
    if n < target_length:
        fbank = torch.cat([fbank, torch.zeros(B, target_length - n, ch, device=fbank.device)], 1)
    elif n > target_length:
        fbank = fbank[:, :target_length, :]
    return fbank[:, :, :-1] if ch % 2 else fbank


def get_mel_from_wav(audio: torch.Tensor, _stft: TacotronSTFT):
    """torch_tools.py:57-61."""
    audio = torch.nan_to_num(torch.clip(audio, -1, 1))
    return _stft.mel_spectrogram(audio)


def wav_to_fbank(waveforms: Sequence[torch.Tensor], target_length: int = 1024, fn_STFT: Optional[TacotronSTFT] = None):
    """torch_tools.py:64-77 after the file decode / resample of read_wav_file (host I/O, not on this path): a list of
    16 kHz mono waveforms -> (fbank (B, target_length, n_mel), log-magnitudes (B, target_length, bins - 1),
    waveform (B, target_length * hop))."""
    assert fn_STFT is not None
    hop = fn_STFT.hop_length
    prepared = []
    for w in waveforms:
        w = pad_wav(normalize_wav(torch.as_tensor(w, dtype=torch.float32)), target_length * hop).unsqueeze(0)
        prepared.append(0.5 * (w / torch.max(torch.abs(w))))
    waveform = torch.cat(prepared, 0)
    fbank, log_mag, _ = get_mel_from_wav(waveform, fn_STFT)
    return (_pad_spec(fbank.transpose(1, 2), target_length), _pad_spec(log_mag.transpose(1, 2), target_length), waveform)
