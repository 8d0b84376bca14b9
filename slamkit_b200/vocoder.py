"""HifiGanB200Vocoder -- the reference's `HiFiGANVocoder` (slamkit/vocoder/hifi_gan_vocoder.py ->
`CodeHiFiGANVocoder`, slamkit/vocoder/hifigan/vocoder.py) on the library's vocoder kernels (`sk_vocoder_*`).

It loads the textlesslib checkpoint layout: `torch.load(model)["generator"]` with weight-norm `weight_g` / `weight_v`
pairs, and the generator's JSON config.  Weight norm is folded on the host in fp64.  `vocode(tokens)` is the
`AudioVocoder` contract: one 1-D unit sequence in, one 1-D device waveform out, with `speaker_id = style_id = 0` and
the duration predictor on when the checkpoint has one, as `HiFiGANVocoder.vocode` calls it.  `vocode_batch` vocodes
many rows in one call; each row's samples are bit-identical to vocoding it alone."""
from __future__ import annotations

import ctypes as C
import json
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib as L


class SkVocoderConfig(C.Structure):
    _fields_ = [
        ("num_embeddings", C.c_int32),
        ("embedding_dim", C.c_int32),
        ("model_in_dim", C.c_int32),
        ("multispkr", C.c_int32),
        ("num_speakers", C.c_int32),
        ("multistyle", C.c_int32),
        ("num_styles", C.c_int32),
        ("upsample_initial_channel", C.c_int32),
        ("n_upsamples", C.c_int32),
        ("upsample_rates", C.c_int32 * 8),
        ("upsample_kernel_sizes", C.c_int32 * 8),
        ("n_resblocks", C.c_int32),
        ("resblock_kernel_sizes", C.c_int32 * 4),
        ("resblock_dilations", (C.c_int32 * 3) * 4),
        ("dur_predictor", C.c_int32),
        ("dur_hidden", C.c_int32),
        ("dur_kernel", C.c_int32),
        ("max_rows", C.c_int32),
        ("max_frames", C.c_int32),
    ]


class SkVocoderConvDesc(C.Structure):
    """sk_vocoder_conv: one convolution layer of the network, run as sk_vocoder_run runs it (see the header)."""
    _fields_ = [
        ("T_in", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32), ("k", C.c_int32),
        ("transposed", C.c_int32), ("rate", C.c_int32), ("dilation", C.c_int32), ("slope", C.c_float),
        ("x", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p), ("valid", C.c_void_p),
        ("up", C.c_int32), ("mode", C.c_int32),
        ("y", C.c_void_p), ("res", C.c_void_p), ("sum", C.c_void_p),
        ("divide", C.c_int32),
        ("prep", C.c_void_p), ("prep_bytes", C.c_int64),
    ]


def parse_config(cfg: Dict) -> Dict:
    """The geometry of a `CodeGenerator` JSON config (generator.py:24-125), or ValueError for what the reference's
    `vocode()` cannot run either (f0 conditioning, `embedder_params`) and for what these kernels do not implement."""
    if cfg.get("f0"):
        raise ValueError("f0-conditioned vocoders are not supported: CodeHiFiGANVocoder.vocode never passes f0")
    if cfg.get("embedder_params"):
        raise ValueError("vocoders with embedder_params are not supported: vocode() passes speaker ids, not embeddings")
    rates, kernels = list(cfg["upsample_rates"]), list(cfg["upsample_kernel_sizes"])
    rk, rd = list(cfg["resblock_kernel_sizes"]), [list(d) for d in cfg["resblock_dilation_sizes"]]
    if len(rates) != len(kernels) or not 1 <= len(rates) <= 8:
        raise ValueError(f"upsample_rates {rates} / upsample_kernel_sizes {kernels}: need 1 to 8 stages of each")
    for u, k in zip(rates, kernels):
        if (k - u) % 2:
            raise ValueError(f"upsample kernel {k} with rate {u}: kernel - rate must be even, so that each stage maps "
                             "L frames to exactly L * rate samples")
    if len(rk) != len(rd) or not 1 <= len(rk) <= 4 or any(len(d) != 3 for d in rd):
        raise ValueError(f"resblock_kernel_sizes {rk} / resblock_dilation_sizes {rd}: need 1 to 4 ResBlocks of 3 dilations")
    E = int(cfg["embedding_dim"])
    spk, sty = bool(cfg.get("multispkr")), bool(cfg.get("multistyle"))
    in_dim = int(cfg.get("model_in_dim", 80))
    if in_dim != E * (1 + spk + sty):
        raise ValueError(f"model_in_dim {in_dim} != embedding_dim {E} x (1 + multispkr + multistyle)")
    dp = cfg.get("dur_predictor_params") or None
    if dp:
        if int(dp["var_pred_kernel_size"]) != 3:
            raise ValueError("var_pred_kernel_size must be 3: the duration predictor's second conv has padding=1 "
                             "hard-coded")
        if int(dp["encoder_embed_dim"]) != E:
            raise ValueError(f"dur_predictor_params.encoder_embed_dim {dp['encoder_embed_dim']} != embedding_dim {E}")
    return dict(num_embeddings=int(cfg["num_embeddings"]), embedding_dim=E, model_in_dim=in_dim, multispkr=spk,
                num_speakers=int(cfg.get("num_speakers", 200)), multistyle=sty, num_styles=int(cfg.get("num_styles", 100)),
                upsample_initial_channel=int(cfg["upsample_initial_channel"]), upsample_rates=rates,
                upsample_kernel_sizes=kernels, resblock_kernel_sizes=rk, resblock_dilation_sizes=rd,
                dur_hidden=int(dp["var_pred_hidden_dim"]) if dp else 0, dur_predictor=bool(dp),
                sampling_rate=int(cfg.get("sampling_rate", 16_000)))


def fold_weight_norm(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """`remove_weight_norm` on a state dict, in fp64: weight = g * v / ||v||, the norm over every dim but dim 0 (for a
    ConvTranspose1d dim 0 is the input channel, so its weight_g is [Cin, 1, 1])."""
    out = {}
    for k, t in state_dict.items():
        if k.endswith(".weight_g"):
            base = k[: -len("_g")]
            v = state_dict[base + "_v"].double()
            g = t.double()
            norm = v.reshape(v.shape[0], -1).norm(dim=1).reshape((-1,) + (1,) * (v.dim() - 1))
            out[base] = (g * v / norm).float()
        elif k.endswith(".weight_v"):
            continue
        else:
            out[k] = t.float()
    return out


class HifiGanB200Vocoder:
    """`CodeHiFiGANVocoder` in eval mode on the GPU.  `max_rows` / `max_frames` size the workspace for one sub-batch;
    larger requests are split into sub-batches of whole rows."""

    def __init__(self, cfg: Dict, state_dict: Dict[str, torch.Tensor], device: str = "cuda:0", max_rows: int = 64,
                 max_frames: int = 16384):
        geo = parse_config(cfg)
        self.cfg = cfg
        self.geometry = geo
        self.lib = L.require_cuda()
        self.dev = torch.device(device)
        torch.cuda.set_device(self.dev)
        c = SkVocoderConfig()
        for name in ("num_embeddings", "embedding_dim", "model_in_dim", "multispkr", "num_speakers", "multistyle",
                     "num_styles", "upsample_initial_channel", "dur_predictor", "dur_hidden"):
            setattr(c, name, int(geo[name]))
        c.n_upsamples = len(geo["upsample_rates"])
        for i, (u, k) in enumerate(zip(geo["upsample_rates"], geo["upsample_kernel_sizes"])):
            c.upsample_rates[i], c.upsample_kernel_sizes[i] = u, k
        c.n_resblocks = len(geo["resblock_kernel_sizes"])
        for j, (k, d) in enumerate(zip(geo["resblock_kernel_sizes"], geo["resblock_dilation_sizes"])):
            c.resblock_kernel_sizes[j] = k
            for a in range(3):
                c.resblock_dilations[j][a] = d[a]
        c.dur_kernel = 3
        c.max_rows, c.max_frames = int(max_rows), int(max_frames)
        self.max_rows, self.max_frames = int(max_rows), int(max_frames)
        self._h = C.c_void_p()
        L.check(self.lib.sk_vocoder_create(C.byref(c), C.byref(self._h)))
        self.upsampling = int(self.lib.sk_vocoder_upsampling(self._h))
        folded = fold_weight_norm(state_dict)
        flat = torch.zeros(int(self.lib.sk_vocoder_param_count(self._h)), dtype=torch.float32)
        buf, off, numel = C.create_string_buffer(64), C.c_int64(), C.c_int64()
        for i in range(self.lib.sk_vocoder_tensor_info(self._h, -1, None, 0, None, None)):
            L.check(self.lib.sk_vocoder_tensor_info(self._h, i, buf, 64, C.byref(off), C.byref(numel)))
            name = buf.value.decode()
            if name not in folded:
                raise KeyError(f"vocoder checkpoint has no '{name}'")
            t = folded[name].reshape(-1)
            if t.numel() != numel.value:
                raise ValueError(f"'{name}' has {t.numel()} elements, the config implies {numel.value}")
            flat[off.value:off.value + numel.value] = t
        self.weights = flat.to(self.dev)
        self.prepared = torch.empty(int(self.lib.sk_vocoder_prepared_bytes(self._h)), dtype=torch.uint8, device=self.dev)
        self.workspace = torch.empty(int(self.lib.sk_vocoder_workspace_bytes(self._h)), dtype=torch.uint8, device=self.dev)
        L.check(self.lib.sk_vocoder_bind(self._h, L.ptr(self.weights), L.ptr(self.prepared), C.c_int64(self.prepared.numel()),
                                         L.ptr(self.workspace), C.c_int64(self.workspace.numel()), L.stream_ptr()))

    @classmethod
    def from_checkpoint(cls, model_path: str, config_path: str, **kw) -> "HifiGanB200Vocoder":
        with open(config_path) as f:
            cfg = json.load(f)
        sd = torch.load(model_path, map_location="cpu", weights_only=True)["generator"]
        return cls(cfg, sd, **kw)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.sk_vocoder_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @property
    def output_sample_rate(self) -> int:
        return self.geometry["sampling_rate"]

    @property
    def device(self) -> torch.device:
        return self.dev

    def to(self, device):
        if torch.device(device) != self.dev:
            raise ValueError(f"this vocoder lives on {self.dev}")
        return self

    # ---- batches ---------------------------------------------------------------------------------------------------
    def _pack(self, codes: Union[torch.Tensor, Sequence[torch.Tensor]], counts: Optional[torch.Tensor]):
        if not isinstance(codes, torch.Tensor):
            rows = [torch.as_tensor(c).reshape(-1) for c in codes]
            n = max([r.numel() for r in rows] + [1])
            packed = torch.full((len(rows), n), -1, dtype=torch.int64)
            for i, r in enumerate(rows):
                packed[i, :r.numel()] = r
            counts = torch.tensor([r.numel() for r in rows], dtype=torch.int32)
            codes = packed
        if codes.dim() == 1:
            codes = codes[None]
        codes = codes.to(self.dev, torch.int64).contiguous()
        if codes.shape[1] == 0:
            codes = torch.full((codes.shape[0], 1), -1, dtype=torch.int64, device=self.dev)
        if counts is None:
            counts = torch.full((codes.shape[0],), codes.shape[1], dtype=torch.int32)
        counts = counts.to(self.dev, torch.int32).contiguous()
        return codes, counts

    def durations(self, codes, counts: Optional[torch.Tensor] = None):
        """Device (dur int32 [B, ld], log_dur fp32 [B, ld], frames int32 [B], status int32 [n_chunks, 2]) of the kept
        units of each row (no synchronisation)."""
        codes, counts = self._pack(codes, counts)
        B, ld = codes.shape
        dur = torch.zeros((B, ld), dtype=torch.int32, device=self.dev)
        logd = torch.zeros((B, ld), dtype=torch.float32, device=self.dev)
        frames = torch.zeros((B,), dtype=torch.int32, device=self.dev)
        chunks = max(1, -(-B // self.max_rows))
        status = torch.zeros((chunks, 2), dtype=torch.int32, device=self.dev)
        for k, b0 in enumerate(range(0, B, self.max_rows)):
            nb = min(self.max_rows, B - b0)
            L.check(self.lib.sk_vocoder_durations(self._h, L.ptr(codes[b0:]), ld, L.ptr(counts[b0:]), nb, L.ptr(dur[b0:]),
                                                  L.ptr(logd[b0:]), L.ptr(frames[b0:]), L.ptr(status[k]), L.stream_ptr()))
        return dur, logd, frames, status

    @torch.inference_mode()
    def vocode_batch(self, codes, counts: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """codes int64 [B, L] (or a list of 1-D sequences) with counts [B] valid entries per row (default: all);
        negative codes are dropped.  Returns (wave fp32 [B, S] on the device, zero past each row's length, lens int64
        [B] on the host).  The host reads the per-row frame counts once, to size `wave`."""
        codes, counts = self._pack(codes, counts)
        B, ld = codes.shape
        _, _, frames, status = self.durations(codes, counts)
        host = torch.cat([frames, status.reshape(-1)]).cpu()
        frames_h, st = host[:B].contiguous(), host[B:].view(-1, 2).sum(0)
        if int(st[0]):
            raise L.SkError(f"{int(st[0])} unit code(s) >= num_embeddings = {self.geometry['num_embeddings']}")
        if int(st[1]) or (B and int(frames_h.max()) > self.max_frames):
            raise L.SkError(f"a row has more frames than this vocoder's max_frames = {self.max_frames}")
        lens = frames_h.long() * self.upsampling
        S = int(lens.max()) if B else 0
        wave = torch.empty((B, S), dtype=torch.float32, device=self.dev)
        if B and S:
            L.check(self.lib.sk_vocoder_run(self._h, L.ptr(codes), ld, L.ptr(counts), B,
                                            frames_h.numpy().ctypes.data_as(C.POINTER(C.c_int32)), L.ptr(wave),
                                            C.c_int64(S), L.stream_ptr()))
        return wave, lens

    def vocode(self, tokens: torch.Tensor, **_) -> torch.Tensor:
        """hifi_gan_vocoder.py:21-22: one unit sequence ([L] or [1, L]) -> 1-D waveform on the device."""
        wave, lens = self.vocode_batch(tokens.reshape(1, -1))
        return wave[0, :int(lens[0])]
