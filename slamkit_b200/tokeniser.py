"""B200UnitTokeniser -- mirror of `slamkit.tokeniser.unit_tokeniser.UnitTokeniser` (slamkit/tokeniser/unit_tokeniser.py:17-121)
for the output contract of hot path (i): run-length dedup, `<Un{i}>` strings, token ids `<PAD>`=0, `<S>`=1,
`<Un{i}>` = i+2 with the `<S> $0 <S>` template.  The dedup runs on the GPU (`sk_rle`) on the device-resident labels; the
string / id mapping is pure host code (no `tokenizers` dependency -- the WordLevel vocab is an affine map).
"""
from __future__ import annotations

import json
import re
from typing import Dict, List, Optional, Union

import numpy as np
import torch

_UNIT_RE = re.compile(r"<Un(\d+)>")


class B200UnitTokeniser:
    def __init__(self, speech_tokeniser=None, dedup: bool = True, bos_eos_token_id: int = 1, pad_token_id: int = 0,
                 num_units: int = 500, load_fe: bool = True):
        self.model = speech_tokeniser if load_fe else None
        self.dedup = dedup
        self.bos_token_id = self.eos_token_id = bos_eos_token_id
        self.pad_token_id = pad_token_id
        self.num_units = num_units
        self.offset = max(self.eos_token_id, self.bos_token_id, self.pad_token_id) + 1   # unit_tokeniser.py:35

    def __len__(self) -> int:     # len(tokeniser.text_tokeniser) in cli/train.py:39-41 -> vocab size 502
        return self.num_units + self.offset

    # ---- path (i) output contract ---------------------------------------------------------------------------------
    def audio_represent(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None) -> List[Dict]:
        """unit_tokeniser.py:54-60: [{'units': (...), 'duration': (...)}] per clip."""
        ids, nf = self.model.units_device(wav, lens)
        if self.dedup:
            units, dur, cnt = self.model.dedup_device(ids, nf)
            u, d, c = units.cpu().numpy(), dur.cpu().numpy(), cnt.cpu().numpy()
            return [{"units": tuple(int(x) for x in u[b, :c[b]]), "duration": tuple(int(x) for x in d[b, :c[b]])}
                    for b in range(u.shape[0])]
        i, n = ids.cpu().numpy(), nf.cpu().numpy()
        return [{"units": i[b, :n[b]], "duration": [1] * int(n[b])} for b in range(i.shape[0])]

    def stringify_representation(self, reps: List[Dict], mode: str = "test") -> List[str]:
        return ["".join(f"<Un{u}>" for u in cur["units"]) for cur in reps]

    def audio_stringify(self, wav, lens=None) -> List[str]:
        return self.stringify_representation(self.audio_represent(wav, lens))

    # ---- path (ii) input contract ---------------------------------------------------------------------------------
    def _encode(self, s: str) -> List[int]:
        units = [int(m) for m in _UNIT_RE.findall(s)]
        return [self.bos_token_id] + [u + self.offset for u in units] + [self.eos_token_id]

    def string_tokenise(self, audio_repr: Union[str, List[str]], padding: bool = False, return_tensors: Optional[str] = None,
                        **_) -> Dict:
        single = isinstance(audio_repr, str)
        seqs = [self._encode(s) for s in ([audio_repr] if single else audio_repr)]
        if padding or return_tensors == "pt":
            n = max(len(s) for s in seqs)
            mask = [[1] * len(s) + [0] * (n - len(s)) for s in seqs]
            seqs = [s + [self.pad_token_id] * (n - len(s)) for s in seqs]
        else:
            mask = [[1] * len(s) for s in seqs]
        if return_tensors == "pt":
            return {"input_ids": torch.tensor(seqs, dtype=torch.int64), "attention_mask": torch.tensor(mask, dtype=torch.int64)}
        if single:
            return {"input_ids": seqs[0], "attention_mask": mask[0]}
        return {"input_ids": seqs, "attention_mask": mask}

    def __call__(self, sample: Union[Dict, str], **kw):
        if isinstance(sample, dict):
            sample = self.stringify_representation([sample])[0]
        return self.string_tokenise(sample, **kw)

    def tokenise(self, wav, lens=None):
        return self.string_tokenise(self.audio_stringify(wav, lens), return_tensors="pt", padding=True)

    @torch.inference_mode()
    def tokenise_device(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None):
        """`tokenise()` without the host strings: unit ids -> dedup (`sk_rle`) -> `[BOS, u + offset..., EOS, PAD...]`
        (`sk_units_to_tokens`), all on the device.  Returns device (ids int64 [B, T], attention_mask int64 [B, T]), equal
        to tokenise()'s.  The host reads the per-row counts once, to size the batch."""
        from . import _lib as L
        fe = self.model
        if fe is None:
            raise RuntimeError("This tokeniser does not have a feature extractor")
        ids, nf = fe.units_device(wav, lens)
        units, counts = ids, nf
        if self.dedup:
            units, _, counts = fe.dedup_device(ids, nf)
        B, T_units = units.shape
        T_out = int(counts.max()) + 2 if B else 2
        out = torch.empty((B, T_out), dtype=torch.int64, device=units.device)
        if B:
            L.check(fe.lib.sk_units_to_tokens(L.ptr(units), L.ptr(counts), B, T_units, self.offset, self.bos_token_id,
                                              self.eos_token_id, self.pad_token_id, L.ptr(out), T_out, L.stream_ptr()))
        mask = (torch.arange(T_out, device=units.device)[None, :] < (counts.long() + 2)[:, None]).long()
        return out, mask

    def prepare_sample(self, sample: dict, **kw):
        return self.string_tokenise(sample["audio_repr"], **kw)

    def decode_sample(self, tokens: torch.Tensor, output_modality: str = "SPEECH") -> torch.Tensor:
        t = tokens[(tokens != self.pad_token_id) & (tokens != self.bos_token_id) & (tokens != self.eos_token_id)]
        return (t - self.offset).to(torch.int64)

    @property
    def fe_sample_rate(self) -> int:
        if self.model is None:
            raise RuntimeError("This tokeniser does not have a feature extractor")
        return self.model.sample_rate

    def save_pretrained(self, save_directory: str, **_):
        with open(f"{save_directory}/tokeniser_config.json", "w") as f:
            json.dump({"dedup": self.dedup, "bos_eos_token_id": self.bos_token_id, "pad_token_id": self.pad_token_id,
                       "num_units": self.num_units, "load_fe": False}, f)

    @classmethod
    def from_pretrained(cls, path: str, **kw) -> "B200UnitTokeniser":
        with open(f"{path}/tokeniser_config.json") as f:
            cfg = json.load(f)
        return cls(speech_tokeniser=None, **cfg, **kw)

    def get_ignore_tokens(self, _=None):
        return None


SPEECH_TOKEN, TEXT_TOKEN = "<speech>", "<text>"


class B200InterleavingTokeniser:
    """Host-side mirror of `slamkit.tokeniser.interleaving_tokeniser.InterleavingTokeniser` for the TRAINING input
    contract of the interleaved speech-text recipe (config/tokeniser/interleaved_hubert_25.yaml, BASELINE cfg-4): an HF
    text tokenizer extended with `<Un0>..<Un{n-1}>`, `<speech>`, `<text>` (interleaving_tokeniser.py:121-127), so the
    model vocabulary is text + units (~152 k rows for Qwen2.5).  `prepare_sample` / `string_tokenise` / `len` are what
    cli/train.py needs; `audio_represent` goes through the same GPU feature extractor as the unit tokeniser.  Building
    the interleaved strings from word alignments (`stringify_representation(mode='train')`) is text-side preprocessing
    outside the hot path (SURVEY.md §2) and is not re-implemented: prepare such token files with the reference."""

    def __init__(self, speech_tokeniser=None, dedup: bool = True, pad_token_id: int = 0, num_units: int = 500,
                 load_fe: bool = True, text_tokeniser_path: str = "facebook/opt-125m", interleave_method: str = "random",
                 interleave_span: Optional[int] = None, interleave_prob: Optional[float] = None):
        from transformers import AutoTokenizer
        self.model = speech_tokeniser if load_fe else None
        self.dedup, self.pad_token_id, self.num_units = dedup, pad_token_id, num_units
        tk = AutoTokenizer.from_pretrained(text_tokeniser_path)
        tk.pad_token_id = pad_token_id
        tk.padding_side = "right"
        tk.add_tokens([f"<Un{x}>" for x in range(num_units)] + [SPEECH_TOKEN, TEXT_TOKEN])
        self.text_tokeniser = tk
        self.interleave_method, self.interleave_span, self.interleave_prob = interleave_method, interleave_span, interleave_prob

    def __len__(self) -> int:
        return len(self.text_tokeniser)

    def audio_represent(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None) -> List[Dict]:
        return B200UnitTokeniser.audio_represent(self, wav, lens)

    def stringify_representation(self, reps: List[Dict], mode: str = "test") -> List[str]:
        if mode == "train":
            raise NotImplementedError("interleaving from word alignments is text-side preprocessing outside the GPU hot "
                                      "path; prepare interleaved token files with the reference's cli/prepare_tokens.py")
        return ["".join(f"<Un{u}>" for u in cur["units"]) for cur in reps]

    def string_tokenise(self, audio_repr, **kw) -> Dict:
        return self.text_tokeniser(audio_repr, add_special_tokens=True, **kw)

    def prepare_sample(self, sample: dict, **kw) -> Dict:
        return self.string_tokenise(sample["audio_repr"], **kw)

    @property
    def fe_sample_rate(self) -> int:
        return B200UnitTokeniser.fe_sample_rate.fget(self)

    def tokenise(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None) -> Dict:
        """interleaving_tokeniser.py:230-233, speech-only batch: `<Un…>` strings through the text tokenizer, right-padded."""
        if not isinstance(wav, torch.Tensor):
            raise NotImplementedError("interleaved (speech + text) inputs are not supported: pass a speech-only wav batch")
        self.text_tokeniser.padding_side = "right"
        strs = self.stringify_representation(self.audio_represent(wav, lens))
        return self.string_tokenise(strs, return_tensors="pt", padding=True)

    def get_ignore_tokens(self, used_token_modality: Optional[str]) -> Optional[List[int]]:
        """interleaving_tokeniser.py:295-310: ids excluded from the log-likelihood.  SPEECH bans every text id except
        bos / eos, plus `<speech>` / `<text>`; TEXT bans the unit ids (not the two markers); anything else bans nothing."""
        tk = self.text_tokeniser
        num_text = len(tk) - self.num_units - 2
        special = [tk.bos_token_id, tk.eos_token_id]
        markers = [tk.encode(SPEECH_TOKEN)[0], tk.encode(TEXT_TOKEN)[0]]
        if used_token_modality and used_token_modality.upper() == "SPEECH":
            return [x for x in range(0, num_text) if x not in special] + markers
        if used_token_modality and used_token_modality.upper() == "TEXT":
            return [x for x in range(num_text, len(tk)) if x not in special + markers]
        return None

    def save_pretrained(self, save_directory: str, **_):
        with open(f"{save_directory}/tokeniser_config.json", "w") as f:
            json.dump({"dedup": self.dedup, "pad_token_id": self.pad_token_id, "num_units": self.num_units, "load_fe": False,
                       "text_tokeniser_path": self.text_tokeniser.name_or_path, "interleave_method": self.interleave_method,
                       "interleave_span": self.interleave_span, "interleave_prob": self.interleave_prob}, f)
