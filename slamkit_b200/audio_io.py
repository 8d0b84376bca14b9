"""Audio file I/O for cli/extract_features.py: PCM WAV via the standard library, FLAC via the library's own decoder
(`sk_flac_*`; the image has no audio backend).  Mirrors what `WavDataset.__getitem__` does after decoding
(cli/extract_features.py:50-57): resample to the target rate if the file's differs (`torchaudio.functional.resample`
defaults: Hann-windowed sinc, lowpass_filter_width 6, rolloff 0.99), THEN average the channels, float32 in [-1, 1)."""
from __future__ import annotations

import math
import struct
import wave
from typing import Tuple

import numpy as np
import torch


def _wav_chunks(path: str):
    """(format tag, channels, sample rate, bits per sample, data offset, data bytes) of a RIFF/WAVE file; the tag of a
    WAVE_FORMAT_EXTENSIBLE file is its sub-format's."""
    with open(path, "rb") as f:
        head = f.read(12)
        if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
            raise ValueError(f"{path}: not a RIFF/WAVE file")
        fmt = None
        while True:
            ch = f.read(8)
            if len(ch) < 8:
                raise ValueError(f"{path}: no data chunk")
            cid, size = ch[:4], struct.unpack("<I", ch[4:])[0]
            if cid == b"fmt ":
                body = f.read(size)
                tag, nch, sr, _, _, bits = struct.unpack("<HHIIHH", body[:16])
                if tag == 0xFFFE and len(body) >= 26:
                    tag = struct.unpack("<H", body[24:26])[0]
                fmt = (tag, nch, sr, bits)
                f.seek(size & 1, 1)
            elif cid == b"data":
                if fmt is None:
                    raise ValueError(f"{path}: data chunk before fmt chunk")
                return fmt + (f.tell(), size)
            else:
                f.seek(size + (size & 1), 1)


def wav_num_frames(path: str) -> int:
    tag, nch, sr, bits, _, size = _wav_chunks(path)
    return size // (nch * bits // 8)


def audio_info(path: str) -> Tuple[int, int]:
    """(frames, sample rate) of a FLAC or WAV file (what torchaudio.info reports as num_frames / sample_rate)."""
    if path.lower().endswith(".flac"):
        i = flac_info(path)
        return i["num_frames"], i["sample_rate"]
    tag, nch, sr, bits, _, size = _wav_chunks(path)
    return size // (nch * bits // 8), sr


def resample(x: torch.Tensor, orig_sr: int, new_sr: int, lowpass_filter_width: int = 6, rolloff: float = 0.99) -> torch.Tensor:
    """Band-limited resampling with the arithmetic of `torchaudio.functional.resample(x, orig_sr, new_sr)` at its default
    arguments (the call at cli/extract_features.py:53-54): reduce the rates by their gcd, build `new` polyphase
    Hann-windowed sinc filters of cutoff `rolloff * min(orig, new)` in float32, run them as a
    stride-`orig` convolution over the zero-padded waveform and keep ceil(new * n / orig) samples.
    x: [..., frames] float32.  Pinned against torchaudio in tests/test_host_cpu.py."""
    if orig_sr == new_sr:
        return x
    g = math.gcd(int(orig_sr), int(new_sr))
    orig, new = int(orig_sr) // g, int(new_sr) // g
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    # torchaudio builds the taps in the waveform's dtype (float32 here), not in float64: for ratios such as 441 -> 160
    # that moves individual taps by ~1e-5, so the restatement keeps float32 throughout
    f32 = torch.float32
    idx = torch.arange(-width, width + orig, dtype=f32)[None, None] / orig
    t = torch.arange(0, -new, -1, dtype=f32)[:, None, None] / new + idx
    t *= base
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    kern = torch.where(t == 0, torch.tensor(1.0, dtype=f32), t.sin() / t)
    kern *= window * (base / orig)                                  # [new, 1, 2*width + orig]
    shape = x.shape
    w = x.reshape(-1, shape[-1]).to(torch.float32)
    n = w.shape[-1]
    w = torch.nn.functional.pad(w, (width, width + orig))
    y = torch.nn.functional.conv1d(w[:, None], kern, stride=orig)   # [rows, new, frames/orig]
    y = y.transpose(1, 2).reshape(w.shape[0], -1)
    target = math.ceil(new * n / orig)
    return y[..., :target].reshape(shape[:-1] + (target,))


def load_wav(path: str, target_sr: int = 16000) -> torch.Tensor:
    tag, ch, sr, bits, off, size = _wav_chunks(path)
    width = bits // 8
    with open(path, "rb") as f:
        f.seek(off)
        raw = f.read(size - size % (ch * width))
    if tag == 3:                                                  # IEEE float, as torchaudio.save writes float32
        if width != 4:
            raise ValueError(f"{path}: unsupported float sample width {width}")
        x = np.frombuffer(raw, dtype="<f4").astype(np.float32)
    elif tag != 1:
        raise ValueError(f"{path}: unsupported WAV format tag {tag}")
    elif width == 2:
        x = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif width == 4:
        x = np.frombuffer(raw, dtype="<i4").astype(np.float32) / 2147483648.0
    elif width == 1:
        x = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    else:
        raise ValueError(f"{path}: unsupported PCM sample width {width}")
    x = torch.from_numpy(x.reshape(-1, ch).T.copy())          # [channels, frames]
    x = resample(x, sr, target_sr)                            # reference order: resample, then the channel mean
    return x.mean(dim=0)


def write_wav(path: str, x: torch.Tensor, sr: int = 16000) -> None:
    pcm = (x.clamp(-1, 1 - 1 / 32768) * 32768.0).round().to(torch.int16).numpy()
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes(pcm.tobytes())


def write_wav_float(path: str, x: torch.Tensor, sr: int = 16000) -> None:
    """Mono 32-bit IEEE-float WAV (format tag 3 with a fact chunk): what torchaudio.save writes for a float32 tensor."""
    data = x.detach().reshape(-1).to("cpu", torch.float32).numpy().astype("<f4").tobytes()
    n = len(data) // 4
    fmt = struct.pack("<HHIIHHH", 3, 1, sr, sr * 4, 4, 32, 0)
    body = (b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"fact" + struct.pack("<II", 4, n)
            + b"data" + struct.pack("<I", len(data)) + data)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


# ---- FLAC through the library's host-side decoder (sk_flac_*) ---------------------------------------------------------
def flac_info(path: str):
    import ctypes as C
    from . import _lib as L
    lib = L.load()
    sr, ch, bps, n = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
    md5 = (C.c_uint8 * 16)()
    L.check(lib.sk_flac_info(path.encode(), C.byref(sr), C.byref(ch), C.byref(bps), C.byref(n), md5))
    return {"sample_rate": sr.value, "channels": ch.value, "bits_per_sample": bps.value, "num_frames": n.value,
            "md5": bytes(md5)}


def flac_decode_int(path: str) -> np.ndarray:
    """Interleaved PCM as int32 [frames, channels]."""
    import ctypes as C
    from . import _lib as L
    lib = L.load()
    info = flac_info(path)
    cap = max(info["num_frames"], 1) + 65536
    buf = np.empty((cap, info["channels"]), dtype=np.int32)
    n = C.c_int64()
    L.check(lib.sk_flac_decode_i32(path.encode(), buf.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(cap), C.byref(n)))
    return buf[:n.value]


def load_flac(path: str, target_sr: int = 16000) -> torch.Tensor:
    """torchaudio.load semantics for integer FLAC: float32 = int / 2^(bits-1), then the channel mean."""
    info = flac_info(path)
    pcm = flac_decode_int(path).astype(np.float32) / float(1 << (info["bits_per_sample"] - 1))
    x = resample(torch.from_numpy(pcm.T.copy()), info["sample_rate"], target_sr)
    return x.mean(dim=0)


def load_audio(path: str, target_sr: int = 16000) -> torch.Tensor:
    return load_flac(path, target_sr) if path.lower().endswith(".flac") else load_wav(path, target_sr)


def audio_num_frames(path: str) -> int:
    return flac_info(path)["num_frames"] if path.lower().endswith(".flac") else wav_num_frames(path)
