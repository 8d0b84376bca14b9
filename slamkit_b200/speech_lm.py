"""B200SpeechLM -- mirror of the reference's `SpeechLM` (slamkit/model/speech_lm.py:8-36) for the modelling metrics:
a trained `B200UnitLM` plus an audio tokeniser, scoring zero-padded waveform batches.

With the unit tokeniser the whole chain runs on the device: HuBERT units (`sk_hubert_units`) -> dedup (`sk_rle`) ->
token ids (`sk_units_to_tokens`) -> LM forward (`sk_lm_forward`) -> per-sequence scores (`sk_seq_loglik`).  The
interleaved tokeniser builds its ids through the text tokenizer on the host, as the reference does."""
from __future__ import annotations

from typing import Optional

import torch


class B200SpeechLM:
    def __init__(self, model, tokeniser, vocoder=None, device: Optional[str] = None):
        if vocoder is not None:
            raise NotImplementedError("vocoding needs a vocoder, which this package does not provide")
        self.model = model
        self.tokeniser = tokeniser
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
        """speech_lm.py:22-36: bf16 [B] log-likelihood of each zero-padded clip (mean over tokens with `mean_nll`)."""
        ids, mask = self.tokenise(wavs, lens)
        ignore = self.tokeniser.get_ignore_tokens(used_token_modality)
        return self.model.sequence_log_likelihood(ids, mean_nll, ignore, attention_mask=mask)
