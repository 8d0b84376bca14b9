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

    def prompt_ids(self, units: torch.Tensor, counts: torch.Tensor) -> Dict[str, torch.Tensor]:
        """The generation prompt of unit_tokeniser.py:75-80 under the left padding SpeechLM.generate sets: row b is
        `[PAD..., BOS, units[b, :counts[b]] + offset]` (the template's EOS dropped), with its attention mask.  Works on
        the tensors' device."""
        B = units.shape[0]
        counts = counts.to(units.device).long()
        T = int(counts.max()) + 1 if B else 1
        col = torch.arange(T, device=units.device)[None, :]
        start = T - 1 - counts[:, None]                                   # column of BOS
        src = (col - start - 1).clamp(0, max(units.shape[1] - 1, 0))
        vals = units.long().gather(1, src) + self.offset if units.shape[1] else torch.zeros_like(src)
        ids = torch.where(col > start, vals, torch.full_like(vals, self.pad_token_id))
        ids = torch.where(col == start, torch.full_like(ids, self.bos_token_id), ids)
        return {"input_ids": ids, "attention_mask": (col >= start).long()}

    @torch.inference_mode()
    def build_prompt(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None,
                     output_modality: Optional[str] = None) -> Dict[str, torch.Tensor]:
        """unit_tokeniser.py:75-80 on the device: HuBERT units -> dedup (`sk_rle`) -> left-padded prompt ids."""
        fe = self.model
        if fe is None:
            raise RuntimeError("This tokeniser does not have a feature extractor")
        ids, nf = fe.units_device(wav, lens)
        if self.dedup:
            ids, _, nf = fe.dedup_device(ids, nf)
        return self.prompt_ids(ids, nf)

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

    def _check_speech_output(self, wav, output_modality: Optional[str]) -> None:
        if not isinstance(wav, torch.Tensor):
            raise NotImplementedError("interleaved (speech + text) inputs are not supported: pass a speech-only wav batch")
        if output_modality is None or output_modality.upper() != "SPEECH":
            raise NotImplementedError(f"output_modality={output_modality!r}: only SPEECH continuations are supported")

    def prompt_layout(self) -> Dict[str, object]:
        """What build_prompt puts around the units, read off the text tokenizer once: `prefix` (the ids it adds before a
        string with add_special_tokens=True: a bos for OPT-style tokenizers, nothing for Qwen2 / NeoX ones), `unit_id` (the
        id of `<Un i>`, i < num_units) and `marker` (the id of `<speech>`).  A trailing eos the tokenizer appends is
        dropped, as interleaving_tokeniser.py:260-262 drops it."""
        lay = self.__dict__.get("_prompt_layout")
        if lay is None:
            tk = self.text_tokeniser
            plain = tk("<Un0>", add_special_tokens=False)["input_ids"]
            full = tk("<Un0>", add_special_tokens=True)["input_ids"]
            at = next((i for i in range(len(full) - len(plain) + 1) if full[i:i + len(plain)] == plain), None)
            if len(plain) != 1 or at is None:
                raise NotImplementedError("the text tokenizer does not encode `<Un0>` as one token")
            suffix = full[at + 1:]
            if suffix and not (len(suffix) == 1 and tk.eos_token_id is not None and suffix[0] == tk.eos_token_id):
                raise NotImplementedError(f"the text tokenizer appends {suffix} after a string; only a trailing eos "
                                          "(dropped) is supported")
            lay = {"prefix": list(full[:at]),
                   "unit_id": tk.convert_tokens_to_ids([f"<Un{u}>" for u in range(self.num_units)]),
                   "marker": tk.convert_tokens_to_ids(SPEECH_TOKEN)}
            self._prompt_layout = lay
        return lay

    def _device_tables(self, device) -> Dict[str, torch.Tensor]:
        key = ("_tables", str(device))
        t = self.__dict__.get(key)
        if t is None:
            lay = self.prompt_layout()
            tk = self.text_tokeniser
            n = len(tk)
            unit_of = torch.full((n,), -1, dtype=torch.long)
            unit_of[torch.tensor(lay["unit_id"], dtype=torch.long)] = torch.arange(self.num_units)
            # decode_sample drops pad / bos / eos and the markers before it looks for units
            drop = [i for i in (tk.pad_token_id, tk.bos_token_id, tk.eos_token_id) if i is not None]
            drop += [tk.encode(SPEECH_TOKEN)[0], tk.encode(TEXT_TOKEN)[0]]
            unit_of[torch.tensor(drop, dtype=torch.long)] = -1
            t = {"unit_id": torch.tensor(lay["unit_id"], dtype=torch.int32, device=device),
                 "prefix": torch.tensor(lay["prefix"] or [0], dtype=torch.int32, device=device),
                 "unit_of": unit_of.to(device)}
            self.__dict__[key] = t
        return t

    def prompt_ids(self, units: torch.Tensor, counts: torch.Tensor) -> Dict[str, torch.Tensor]:
        """The SPEECH generation prompt of interleaving_tokeniser.py:242-263, left-padded as SpeechLM.generate pads it,
        from sk_rle's units int32 [B, T_units] and counts int32 [B] (device): row b is
        `[pad..., prefix..., <Un u>..., <speech>]` with its attention mask (`sk_units_to_prompt`)."""
        from . import _lib as L
        lay, tab = self.prompt_layout(), self._device_tables(units.device)
        B, T_units = units.shape
        units, counts = units.to(torch.int32).contiguous(), counts.to(units.device, torch.int32).contiguous()
        T = len(lay["prefix"]) + (int(counts.max()) if B else 0) + 1
        ids = torch.empty((B, T), dtype=torch.int64, device=units.device)
        mask = torch.empty_like(ids)
        if B:
            L.check(L.load().sk_units_to_prompt(L.ptr(units), L.ptr(counts), B, T_units, L.ptr(tab["unit_id"]),
                                                self.num_units, L.ptr(tab["prefix"]), len(lay["prefix"]),
                                                int(lay["marker"]), int(self.text_tokeniser.pad_token_id), L.ptr(ids),
                                                L.ptr(mask), T, L.stream_ptr()))
        return {"input_ids": ids, "attention_mask": mask}

    @torch.inference_mode()
    def build_prompt(self, wav: torch.Tensor, lens: Optional[torch.Tensor] = None,
                     output_modality: Optional[str] = "SPEECH") -> Dict[str, torch.Tensor]:
        """interleaving_tokeniser.py:242-263 for a speech-only batch and SPEECH output, on the device: HuBERT units ->
        dedup (`sk_rle`) -> left-padded `[prefix, <Un u>..., <speech>]` rows."""
        self._check_speech_output(wav, output_modality)
        fe = self.model
        if fe is None:
            raise RuntimeError("This tokeniser does not have a feature extractor")
        ids, nf = fe.units_device(wav, lens)
        if self.dedup:
            ids, _, nf = fe.dedup_device(ids, nf)
        return self.prompt_ids(ids, nf)

    def allowed_ids(self, output_modality: str = "SPEECH", vocab_size: Optional[int] = None) -> List[int]:
        """The ids a SPEECH continuation may emit: the complement of get_ignore_tokens('SPEECH') in a model vocabulary
        of `vocab_size` ids (default: the tokenizer's): the units, the tokenizer's bos / eos, whatever the reference's ban
        list leaves, and the model's ids past the tokenizer's, which the ban list does not cover."""
        if output_modality is None or output_modality.upper() != "SPEECH":
            raise NotImplementedError(f"output_modality={output_modality!r}: only SPEECH continuations are supported")
        ban = set(self.get_ignore_tokens("SPEECH"))
        n = len(self.text_tokeniser) if vocab_size is None else int(vocab_size)
        return [i for i in range(n) if i not in ban]

    def decode_units(self, tokens: torch.Tensor) -> torch.Tensor:
        """Batched device form of decode_sample(·, 'SPEECH'): the unit index of every `<Un i>` id of tokens [N, T],
        -1 elsewhere (pad, bos, eos, markers, text and ids outside the tokenizer).  `vocode_batch` drops the -1s."""
        unit_of = self._device_tables(tokens.device)["unit_of"]
        t = tokens.long()
        ok = (t >= 0) & (t < unit_of.numel())
        return torch.where(ok, unit_of[t.clamp(0, unit_of.numel() - 1)], torch.full_like(t, -1))

    def decode_sample(self, tokens: torch.Tensor, output_modality: str = "SPEECH") -> torch.Tensor:
        """interleaving_tokeniser.py:268-287 for SPEECH: the `<Un i>` units of tokens, in order."""
        if output_modality is None or output_modality.upper() != "SPEECH":
            raise NotImplementedError(f"output_modality={output_modality!r}: only SPEECH continuations are supported")
        u = self.decode_units(tokens.reshape(-1))
        return u[u >= 0]

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
