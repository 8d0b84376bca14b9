"""HubertB200FeatureExtractor -- host-side mirror of the reference's AudioFeatureExtractor plugin for hot path (i).

Mirrors `slamkit.feature_extractor.hubert_feature_extractor.HubertFeatureExtractor`
(slamkit/feature_extractor/hubert_feature_extractor.py:16-57) behind the ABC of
slamkit/feature_extractor/audio_feature_extractor.py:7-30: `extract(wav, lens) -> List[np.ndarray]`,
`get_unit_duration()`, `sample_rate`.  Selected with `feature_extractor_type: hubert_b200`
(slamkit/tokeniser/audio_tokeniser.py:99-104 dispatches on that string).  All compute -- conv encoder, transformer,
k-means argmin, length trim -- runs in libslamkit_b200.so (`sk_hubert_*`); only int32 labels come back to the host.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L

GROUP_PAD = 64


@dataclass
class HubertB200Config:
    """mHuBERT-25Hz geometry (config/tokeniser/feature_extractor/mhubert_25.yaml; conv stack per SURVEY.md §4)."""
    conv_dim: int = 512
    conv_kernel: Tuple[int, ...] = (10, 3, 3, 3, 3, 2, 2, 2)
    conv_stride: Tuple[int, ...] = (5, 2, 2, 2, 2, 2, 2, 2)
    hidden: int = 768
    n_heads: int = 12
    ffn: int = 3072
    layer: int = 11                 # hidden_states[layer] -> `layer` encoder layers are executed
    pos_conv_kernel: int = 128
    pos_conv_groups: int = 16
    n_units: int = 500
    ln_eps: float = 1e-5
    pad: int = 40

    @staticmethod
    def from_hf(cfg, layer: int, n_units: int) -> "HubertB200Config":
        return HubertB200Config(conv_dim=cfg.conv_dim[0], conv_kernel=tuple(cfg.conv_kernel),
                                conv_stride=tuple(cfg.conv_stride), hidden=cfg.hidden_size,
                                n_heads=cfg.num_attention_heads, ffn=cfg.intermediate_size, layer=layer,
                                pos_conv_kernel=cfg.num_conv_pos_embeddings,
                                pos_conv_groups=cfg.num_conv_pos_embedding_groups, n_units=n_units,
                                ln_eps=cfg.layer_norm_eps)


def prepare_weights(p: Dict[str, torch.Tensor], cfg: HubertB200Config) -> Dict[str, torch.Tensor]:
    """Reference-named fp32 parameters (the names of oracle/hubert_oracle.init_hubert_params, see `from_hf_state_dict`)
    -> the prepared layout the C ABI expects (include/slamkit_b200.h, sk_hubert_tensor_info)."""
    Cc, H, G, K = cfg.conv_dim, cfg.hidden, cfg.pos_conv_groups, cfg.pos_conv_kernel
    cg = H // G
    out: Dict[str, torch.Tensor] = {}
    out["conv0.w"] = p["conv0.weight"].reshape(Cc, cfg.conv_kernel[0])
    out["gn.g"], out["gn.b"] = p["gn.weight"], p["gn.bias"]
    for i in range(1, len(cfg.conv_kernel)):
        # [co, ci, j] -> [co, j*C + ci]: a window of k consecutive channels-last frames is one contiguous row
        out[f"conv{i}.w"] = p[f"conv{i}.weight"].permute(0, 2, 1).reshape(Cc, cfg.conv_kernel[i] * Cc)
    out["fp.ln.g"], out["fp.ln.b"] = p["fp.ln.weight"], p["fp.ln.bias"]
    out["fp.w"], out["fp.b"] = p["fp.proj.weight"], p["fp.proj.bias"]
    v = p["pos.v"].double()
    w = (p["pos.g"].double() * v / v.norm(dim=(0, 1), keepdim=True)).float()      # torch weight_norm(dim=2), folded
    wp = torch.zeros(G, GROUP_PAD, K, GROUP_PAD)
    wp[:, :cg, :, :cg] = w.view(G, cg, cg, K).permute(0, 1, 3, 2)                  # [g, co, j, ci]
    out["pos.w"] = wp.reshape(G * GROUP_PAD, K * GROUP_PAD)
    bp = torch.zeros(G, GROUP_PAD)
    bp[:, :cg] = p["pos.bias"].view(G, cg)
    out["pos.b"] = bp.reshape(-1)
    out["enc.ln.g"], out["enc.ln.b"] = p["enc.ln.weight"], p["enc.ln.bias"]
    for l in range(cfg.layer):
        q = f"layers.{l}."
        out[q + "wqkv"] = torch.cat([p[q + "q.weight"], p[q + "k.weight"], p[q + "v.weight"]], 0)
        out[q + "bqkv"] = torch.cat([p[q + "q.bias"], p[q + "k.bias"], p[q + "v.bias"]], 0)
        out[q + "wo"], out[q + "bo"] = p[q + "o.weight"], p[q + "o.bias"]
        out[q + "ln1.g"], out[q + "ln1.b"] = p[q + "ln1.weight"], p[q + "ln1.bias"]
        out[q + "ff1.w"], out[q + "ff1.b"] = p[q + "ff1.weight"], p[q + "ff1.bias"]
        out[q + "ff2.w"], out[q + "ff2.b"] = p[q + "ff2.weight"], p[q + "ff2.bias"]
        out[q + "ln2.g"], out[q + "ln2.b"] = p[q + "ln2.weight"], p[q + "ln2.bias"]
    U = cfg.n_units
    Up = (U + 63) // 64 * 64
    km = torch.zeros(Up, H)
    km[:U] = p["kmeans.centers"]
    out["km.centers"] = km
    return out


def from_hf_state_dict(sd: Dict[str, torch.Tensor], centers: np.ndarray, cfg: HubertB200Config) -> Dict[str, torch.Tensor]:
    """HF `HubertModel.state_dict()` + sklearn `cluster_centers_` -> the reference-style parameter names used above."""
    p = {"conv0.weight": sd["feature_extractor.conv_layers.0.conv.weight"],
         "gn.weight": sd["feature_extractor.conv_layers.0.layer_norm.weight"],
         "gn.bias": sd["feature_extractor.conv_layers.0.layer_norm.bias"]}
    for i in range(1, len(cfg.conv_kernel)):
        p[f"conv{i}.weight"] = sd[f"feature_extractor.conv_layers.{i}.conv.weight"]
    p["fp.ln.weight"], p["fp.ln.bias"] = sd["feature_projection.layer_norm.weight"], sd["feature_projection.layer_norm.bias"]
    p["fp.proj.weight"], p["fp.proj.bias"] = sd["feature_projection.projection.weight"], sd["feature_projection.projection.bias"]
    p["pos.bias"] = sd["encoder.pos_conv_embed.conv.bias"]
    if "encoder.pos_conv_embed.conv.parametrizations.weight.original0" in sd:
        p["pos.g"] = sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"]
        p["pos.v"] = sd["encoder.pos_conv_embed.conv.parametrizations.weight.original1"]
    else:
        p["pos.g"], p["pos.v"] = sd["encoder.pos_conv_embed.conv.weight_g"], sd["encoder.pos_conv_embed.conv.weight_v"]
    p["enc.ln.weight"], p["enc.ln.bias"] = sd["encoder.layer_norm.weight"], sd["encoder.layer_norm.bias"]
    for l in range(cfg.layer):
        q, h = f"layers.{l}.", f"encoder.layers.{l}."
        for a, b in (("q", "attention.q_proj"), ("k", "attention.k_proj"), ("v", "attention.v_proj"),
                     ("o", "attention.out_proj"), ("ff1", "feed_forward.intermediate_dense"),
                     ("ff2", "feed_forward.output_dense"), ("ln1", "layer_norm"), ("ln2", "final_layer_norm")):
            p[q + a + ".weight"], p[q + a + ".bias"] = sd[h + b + ".weight"], sd[h + b + ".bias"]
    p["kmeans.centers"] = torch.from_numpy(np.asarray(centers, dtype=np.float32))
    return {k: v.detach().float() for k, v in p.items()}


def random_params(cfg: HubertB200Config, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded random weights in the reference's parameter naming (synthetic benchmarks / smoke tests: no pretrained
    mHuBERT checkpoint is reachable offline)."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std=1.0):
        return torch.randn(shape, generator=g) * std

    Cc, H, Fd, K, G = cfg.conv_dim, cfg.hidden, cfg.ffn, cfg.pos_conv_kernel, cfg.pos_conv_groups
    p = {"conv0.weight": rn(Cc, 1, cfg.conv_kernel[0], std=math.sqrt(2.0 / cfg.conv_kernel[0])),
         "gn.weight": 1.0 + 0.1 * rn(Cc), "gn.bias": 0.1 * rn(Cc)}
    for i in range(1, len(cfg.conv_kernel)):
        p[f"conv{i}.weight"] = rn(Cc, Cc, cfg.conv_kernel[i], std=math.sqrt(2.0 / (Cc * cfg.conv_kernel[i])))
    p["fp.ln.weight"], p["fp.ln.bias"] = 1.0 + 0.1 * rn(Cc), 0.1 * rn(Cc)
    p["fp.proj.weight"], p["fp.proj.bias"] = rn(H, Cc, std=1.0 / math.sqrt(Cc)), 0.02 * rn(H)
    p["pos.v"] = rn(H, H // G, K, std=math.sqrt(4.0 / (K * H)))
    p["pos.g"] = p["pos.v"].norm(dim=(0, 1), keepdim=True)
    p["pos.bias"] = 0.02 * rn(H)
    p["enc.ln.weight"], p["enc.ln.bias"] = 1.0 + 0.1 * rn(H), 0.1 * rn(H)
    for l in range(cfg.layer):
        q = f"layers.{l}."
        for nm in ("q", "k", "v", "o"):
            p[q + nm + ".weight"], p[q + nm + ".bias"] = rn(H, H, std=1.0 / math.sqrt(H)), 0.02 * rn(H)
        p[q + "ln1.weight"], p[q + "ln1.bias"] = 1.0 + 0.1 * rn(H), 0.1 * rn(H)
        p[q + "ff1.weight"], p[q + "ff1.bias"] = rn(Fd, H, std=1.0 / math.sqrt(H)), 0.02 * rn(Fd)
        p[q + "ff2.weight"], p[q + "ff2.bias"] = rn(H, Fd, std=1.0 / math.sqrt(Fd)), 0.02 * rn(H)
        p[q + "ln2.weight"], p[q + "ln2.bias"] = 1.0 + 0.1 * rn(H), 0.1 * rn(H)
    p["kmeans.centers"] = rn(cfg.n_units, H)
    return p


class HubertB200FeatureExtractor(torch.nn.Module):
    """Drop-in for `HubertFeatureExtractor` (same constructor keys via `from_pretrained_args`, same `extract` contract)."""

    def __init__(self, config: HubertB200Config, params: Optional[Dict[str, torch.Tensor]] = None,
                 device: str = "cuda:0", max_batch: int = 64, max_samples: int = 480000, load_config_only: bool = False):
        super().__init__()
        self.config = config
        self.layer, self.num_units = config.layer, config.n_units
        self._h = None
        if load_config_only:          # hubert_feature_extractor.py:28-30: usable for get_unit_duration() without weights
            return
        assert params is not None, "weights are required unless load_config_only=True"
        self.lib = L.require_cuda()
        self.dev = torch.device(device)
        torch.cuda.set_device(self.dev)
        ck = (C.c_int32 * 8)(*(list(config.conv_kernel) + [0] * (8 - len(config.conv_kernel))))
        cs = (C.c_int32 * 8)(*(list(config.conv_stride) + [0] * (8 - len(config.conv_stride))))
        c = L.SkHubertConfig(len(config.conv_kernel), config.conv_dim, ck, cs, config.hidden, config.n_heads, config.ffn,
                             config.layer, config.pos_conv_kernel, config.pos_conv_groups, config.n_units, config.ln_eps,
                             config.pad)
        self._h = C.c_void_p()
        L.check(self.lib.sk_hubert_create(C.byref(c), C.byref(self._h)))
        n = int(self.lib.sk_hubert_param_count(self._h))
        flat = torch.zeros(n, dtype=torch.float32)
        prepared = prepare_weights(params, config)
        nt = self.lib.sk_hubert_tensor_info(self._h, -1, None, 0, None, None, None)
        buf = C.create_string_buffer(64)
        for i in range(nt):
            off, r, cc = C.c_int64(), C.c_int32(), C.c_int32()
            L.check(self.lib.sk_hubert_tensor_info(self._h, i, buf, 64, C.byref(off), C.byref(r), C.byref(cc)))
            t = prepared[buf.value.decode()].reshape(-1).float()
            assert t.numel() == r.value * cc.value, (buf.value, t.shape, r.value, cc.value)
            flat[off.value:off.value + t.numel()] = t
        self.weights = flat.to(self.dev)
        self.prepared = torch.empty(int(self.lib.sk_hubert_prepared_bytes(self._h)), dtype=torch.uint8, device=self.dev)
        self.workspace = None
        self._bind(max_batch, max_samples)

    def _bind(self, B: int, S: int) -> None:
        need = int(self.lib.sk_hubert_workspace_bytes(self._h, B, S))
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.dev)
        L.check(self.lib.sk_hubert_bind(self._h, L.ptr(self.weights), L.ptr(self.prepared),
                                        C.c_int64(self.prepared.numel()), L.ptr(self.workspace),
                                        C.c_int64(self.workspace.numel()), L.stream_ptr()))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.sk_hubert_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- the AudioFeatureExtractor contract ---------------------------------------------------------------------
    def frames(self, n_samples: int) -> int:
        return int(self.lib.sk_hubert_frames(self._h, n_samples))

    def units_device(self, wav: torch.Tensor, lens: Optional[torch.Tensor]):
        """Device-resident result: (ids int32 [B,T], n_frames int32 [B])."""
        assert wav.dim() == 2
        B, S = wav.shape
        if int(self.lib.sk_hubert_workspace_bytes(self._h, B, S)) > self.workspace.numel():
            self._bind(B, S)
        w = wav.to(self.dev, dtype=torch.float32, non_blocking=True).contiguous()
        ln = lens.to(self.dev, dtype=torch.int64, non_blocking=True).contiguous() if lens is not None else None
        T = self.frames(S)
        ids = torch.empty((B, T), dtype=torch.int32, device=self.dev)
        nf = torch.empty((B,), dtype=torch.int32, device=self.dev)
        L.check(self.lib.sk_hubert_units(self._h, L.ptr(w), L.ptr(ln), B, S, L.ptr(ids), L.ptr(nf), L.stream_ptr()))
        return ids, nf

    @torch.inference_mode()
    def extract(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None) -> List[np.ndarray]:
        """hubert_feature_extractor.py:40-50: list of per-clip unit-id arrays, trimmed to ceil(len/S*T) frames.
        Raises ValueError when the audio holds NaN or Inf, as the reference's k-means input validation does (the
        device labels of such clips are in range but meaningless)."""
        ids, nf = self.units_device(wav, lens)
        finite = bool(torch.isfinite(wav).all())
        ids_h, nf_h = ids.cpu().numpy(), nf.cpu().numpy()
        if not finite:
            raise ValueError("HuBERT features are not finite: the input audio holds NaN or Inf samples")
        return [ids_h[b, :nf_h[b]] for b in range(ids_h.shape[0])]

    @torch.inference_mode()
    def features(self, wav: torch.Tensor) -> torch.Tensor:
        """fp32 hidden_states[layer] ([B,T,hidden]) -- for parity checks only."""
        B, S = wav.shape
        if int(self.lib.sk_hubert_workspace_bytes(self._h, B, S)) > self.workspace.numel():
            self._bind(B, S)
        w = wav.to(self.dev, dtype=torch.float32).contiguous()
        T = self.frames(S)
        feat = torch.empty((B * T, self.config.hidden), dtype=torch.float32, device=self.dev)
        L.check(self.lib.sk_hubert_features(self._h, L.ptr(w), B, S, L.ptr(feat), L.stream_ptr()))
        return feat.view(B, T, -1)

    @torch.inference_mode()
    def debug_stage(self, wav: torch.Tensor, stage: int, rows: int, cols: int) -> torch.Tensor:
        """Test hook (sk_hubert_debug_stage): fp32 tensor of one intermediate stage, shape [rows, cols]."""
        B, S = wav.shape
        if int(self.lib.sk_hubert_workspace_bytes(self._h, B, S)) > self.workspace.numel():
            self._bind(B, S)
        w = wav.to(self.dev, dtype=torch.float32).contiguous()
        out = torch.empty((rows, cols), dtype=torch.float32, device=self.dev)
        L.check(self.lib.sk_hubert_debug_stage(self._h, L.ptr(w), B, S, int(stage), L.ptr(out), L.stream_ptr()))
        return out

    def dedup_device(self, ids: torch.Tensor, n_frames: torch.Tensor):
        """Run-length dedup on the GPU (UnitTokeniser.audio_represent, unit_tokeniser.py:57)."""
        B, T = ids.shape
        units, dur = torch.empty_like(ids), torch.empty_like(ids)
        cnt = torch.empty((B,), dtype=torch.int32, device=ids.device)
        L.check(self.lib.sk_rle(L.ptr(ids), L.ptr(n_frames), L.ptr(units), L.ptr(dur), L.ptr(cnt), B, T, L.stream_ptr()))
        return units, dur, cnt

    def get_unit_duration(self) -> float:
        return math.prod(self.config.conv_stride) / self.sample_rate

    @property
    def sample_rate(self) -> int:
        return 16_000
