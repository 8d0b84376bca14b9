"""B200SpeechLM -- mirror of the reference's `SpeechLM` (slamkit/model/speech_lm.py:8-63): a trained `B200UnitLM` plus
an audio tokeniser and, optionally, a unit vocoder, scoring and continuing zero-padded waveform batches.

With the unit tokeniser the whole chain runs on the device: HuBERT units (`sk_hubert_units`) -> dedup (`sk_rle`) ->
token ids (`sk_units_to_tokens`) -> LM forward (`sk_lm_forward`) -> per-sequence scores (`sk_seq_loglik`).  `generate`
continues left-padded prompts with the cached decoder and vocodes every row in one batched `sk_vocoder_run` call.  The
interleaved tokeniser scores through the text tokenizer on the host, as the reference does; it continues speech on the
device: `sk_units_to_prompt` builds the prompts and the decode steps compute only the head rows of the ids a SPEECH
continuation may emit (`allowed_token_ids`)."""
from __future__ import annotations

from typing import List, Optional

import torch


class B200SpeechLM:
    def __init__(self, model, tokeniser, vocoder=None, device: Optional[str] = None):
        self.model = model
        self.tokeniser = tokeniser
        self.vocoder = vocoder
        self.device = torch.device(device) if device is not None else model.device

    def tokenise(self, wavs: torch.Tensor, lens: Optional[torch.Tensor] = None):
        """(ids int64 [B, T], attention_mask [B, T]), right-padded; on the device for the unit tokeniser."""
        if hasattr(self.tokeniser, "tokenise_device"):
            return self.tokeniser.tokenise_device(wavs, lens)
        enc = self.tokeniser.tokenise(wavs, lens)
        return enc["input_ids"], enc["attention_mask"]

    @torch.inference_mode()
    def log_likelihood(self, wavs: torch.Tensor, lens: Optional[torch.Tensor] = None, mean_nll: bool = True,
                       used_token_modality: Optional[str] = None) -> torch.Tensor:
        """speech_lm.py:22-36: [B] log-likelihood of each zero-padded clip (mean over tokens with `mean_nll`), in the model's
        precision (bf16, or fp32 for an fp32 inference model)."""
        ids, mask = self.tokenise(wavs, lens)
        ignore = self.tokeniser.get_ignore_tokens(used_token_modality)
        return self.model.sequence_log_likelihood(ids, mean_nll, ignore, attention_mask=mask)

    @torch.inference_mode()
    def generate(self, wavs: torch.Tensor, lens: Optional[torch.Tensor] = None, output_modality: str = "SPEECH",
                 remove_prompt: bool = False, **kwargs) -> List[torch.Tensor]:
        """speech_lm.py:38-55: continue each zero-padded prompt clip; with a vocoder, one waveform per row (an empty
        tensor for an empty continuation), otherwise the decoded unit ids.  With `num_return_sequences = k` there are
        B*k rows, the k continuations of each prompt adjacent (HF's order)."""
        if not hasattr(self.tokeniser, "build_prompt"):
            raise NotImplementedError(f"generate: {type(self.tokeniser).__name__} cannot build generation prompts "
                                      "(build_prompt); use the unit or the interleaved tokeniser")
        if output_modality is None or output_modality.upper() != "SPEECH":
            raise NotImplementedError(f"output_modality={output_modality!r}: only SPEECH continuations are supported")
        tokens = self.tokeniser.build_prompt(wavs, lens, output_modality=output_modality)
        if hasattr(self.tokeniser, "allowed_ids"):
            # the reference bans every id of get_ignore_tokens; the same continuation from the allowed ids' head rows
            kwargs["allowed_token_ids"] = self.tokeniser.allowed_ids(output_modality, self.model.config.vocab_size)
        else:
            ignore = self.tokeniser.get_ignore_tokens(output_modality)
            kwargs["bad_words_ids"] = [[tok] for tok in ignore] if ignore is not None else None
        conts = self.model.generate(tokens["input_ids"], attention_mask=tokens["attention_mask"], **kwargs)
        if remove_prompt:
            conts = conts[..., tokens["input_ids"].size(1):]
        if hasattr(self.tokeniser, "decode_units") and self.vocoder is not None:
            wave, wl = self.vocoder.vocode_batch(self.tokeniser.decode_units(conts))
            return [wave[i, :int(wl[i])] if int(wl[i]) > 0 else torch.zeros(0, device=wave.device)
                    for i in range(conts.shape[0])]
        decoded = [self.tokeniser.decode_sample(c, output_modality=output_modality) for c in conts]
        if self.vocoder is None:
            return decoded
        wave, wl = self.vocoder.vocode_batch(decoded)
        return [wave[i, :int(wl[i])] if int(wl[i]) > 0 else torch.zeros(0, device=wave.device)
                for i in range(len(decoded))]
