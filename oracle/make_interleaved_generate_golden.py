"""Generate tests/golden/interleaved_generate_tiny.npz by running the REFERENCE's interleaved speech continuation on the
CPU: `InterleavingTokeniser.build_prompt` / `get_ignore_tokens` / `decode_sample`
(slamkit/tokeniser/interleaving_tokeniser.py) and HF `generate` with the SPEECH ban list as `bad_words_ids`, the calls
`SpeechLM.generate` (slamkit/model/speech_lm.py:38-55) makes.

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_interleaved_generate_golden.py`); the fixture is
committed and is what tests/test_interleaved_generate_cpu.py and tests/test_gpu_interleaved_generate.py compare against.
The reference does not exist on the GPU box, so nothing at test time imports it; the tests rebuild the two text
tokenizers with `text_tokeniser` below, which needs only `tokenizers` / `transformers`.

What is pinned, for a WordLevel text tokenizer with a bos prefix (tag "bos", OPT-style) and one without ("nobos",
Qwen2-style), each extended with 500 `<Un i>` ids and `<speech>` / `<text>`:
  <tag>_prompt_ids / _mask   build_prompt of four unit rows (empty, 1 unit, ragged), left-padded as SpeechLM pads
  <tag>_allowed              the complement of get_ignore_tokens('SPEECH') in the tokenizer's vocabulary
  <tag>_unit_id / _marker / _prefix   the `<Un i>` ids, the `<speech>` id and the ids put before a string
  <tag>_out                  HF greedy generate (6 new tokens, eos = the tokenizer's, pad 0) of a tiny seeded bf16
                             Qwen2ForCausalLM (vocab = len(tokenizer), weights = oracle.lm_oracle.init_params(seed 19,
                             std 0.2)) on the prompts, with the ban list as bad_words_ids.  Every greedy choice of HF's
                             bf16 model is also the fp32 model's and wins by at least MARGIN over the runner-up among
                             the allowed ids, so a different bf16 summation order does not flip it
  <tag>_units / _units_len   decode_sample(row, 'SPEECH') of every output row (prompt included), packed
  units / units_len          the four unit rows
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UNITS = [[], [7], [3, 499, 0, 12, 250], [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
NUM_UNITS, NEW, STD = 500, 6, 0.2
SEED = 19           # the first seed from 7 on whose greedy steps all win by >= MARGIN in fp32 (see _min_margin)
MARGIN = 0.05
MODEL = dict(hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256)


def text_tokeniser(path: str, bos: bool) -> str:
    """A local WordLevel text tokenizer saved to `path` (bos prefix or none, eos `</s>`, pad `<pad>` = 0)."""
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from transformers import PreTrainedTokenizerFast
    vocab = {"<pad>": 0, "<s>": 1, "</s>": 2, "hello": 3, "world": 4, "<unk>": 5}
    tk = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    if bos:
        tk.post_processor = processors.TemplateProcessing(single="<s> $A", special_tokens=[("<s>", 1)])
    PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>", pad_token="<pad>", bos_token="<s>" if bos else None,
                            eos_token="</s>").save_pretrained(path)
    return path


def _qwen2(vocab: int):
    from transformers import Qwen2Config, Qwen2ForCausalLM
    from oracle.lm_oracle import OracleLMConfig, init_params
    c = OracleLMConfig(vocab_size=vocab, **MODEL)
    sd = {k[len("lm."):]: v for k, v in init_params(c, seed=SEED, std=STD).items()}
    cfg = Qwen2Config(vocab_size=vocab, hidden_size=c.hidden, intermediate_size=c.ffn, num_hidden_layers=c.n_layers,
                      num_attention_heads=c.n_heads, num_key_value_heads=c.n_kv_heads, max_position_embeddings=256,
                      rms_norm_eps=c.rms_eps, rope_theta=c.rope_theta, tie_word_embeddings=True, torch_dtype="bfloat16")
    m = Qwen2ForCausalLM(cfg).to(torch.bfloat16).eval()
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("lm_head" in k for k in missing), (missing, unexpected)
    m.tie_weights()
    return m


def _min_margin(model, gen, prompt_mask, ignore) -> float:
    """Smallest fp32 gap between the logit of the token HF's bf16 greedy step chose and the best other allowed logit, over
    the generated steps of rows that have not finished (negative if the fp32 model would choose another token)."""
    prompt_len = prompt_mask.shape[1]
    mask = torch.cat([prompt_mask, torch.ones(gen.shape[0], gen.shape[1] - prompt_len, dtype=prompt_mask.dtype)], 1)
    with torch.inference_mode():
        logits = model.float()(gen, attention_mask=mask).logits
    logits = torch.tensor(logits.numpy())               # a normal tensor, writable outside inference mode
    model.to(torch.bfloat16)
    logits[..., ignore] = float("-inf")
    worst = float("inf")
    for r in range(gen.shape[0]):
        for t in range(prompt_len, gen.shape[1]):
            if t > prompt_len and int(gen[r, t - 1]) == 2:
                break
            row = logits[r, t - 1].clone()
            chosen = float(row[int(gen[r, t])])
            row[int(gen[r, t])] = float("-inf")
            worst = min(worst, chosen - float(row.max()))      # negative: fp32 would choose another token
    return worst


def main(out_path: str):
    sys.path.insert(0, "/root/reference")
    from oracle.make_goldens import _stub_omegaconf
    try:
        import omegaconf  # noqa: F401
    except ImportError:
        _stub_omegaconf()
    from slamkit.tokeniser.interleaving_tokeniser import InterleavingTokeniser

    out = {"units": np.array([u for r in UNITS for u in r], np.int64), "units_len": np.array([len(r) for r in UNITS])}
    reps = [{"units": tuple(r), "duration": tuple([1] * len(r))} for r in UNITS]
    tmp = tempfile.mkdtemp()
    for tag, bos in (("bos", True), ("nobos", False)):
        it = InterleavingTokeniser(None, num_units=NUM_UNITS, load_fe=False,
                                   text_tokeniser_path=text_tokeniser(os.path.join(tmp, tag), bos))
        it.audio_represent = lambda wav, lens=None: reps            # the units, as the feature extractor would give them
        tk = it.text_tokeniser
        tk.padding_side = "left"                                  # as SpeechLM.generate sets it
        prompt = it.build_prompt(torch.zeros(len(UNITS), 16), output_modality="SPEECH")
        ignore = it.get_ignore_tokens("SPEECH")
        ban = set(ignore)
        model = _qwen2(len(tk))
        with torch.inference_mode():
            gen = model.generate(prompt["input_ids"], attention_mask=prompt["attention_mask"], do_sample=False,
                                 max_new_tokens=NEW, bad_words_ids=[[i] for i in ignore], eos_token_id=tk.eos_token_id,
                                 pad_token_id=0)
        margin = _min_margin(model, gen, prompt["attention_mask"], ignore)
        assert margin >= MARGIN, f"{tag}: a greedy step wins by only {margin:.4f}; pick another SEED"
        print(tag, "smallest greedy margin", margin)
        dec = [it.decode_sample(row, "SPEECH") for row in gen]
        out.update({
            f"{tag}_prompt_ids": prompt["input_ids"].numpy(), f"{tag}_prompt_mask": prompt["attention_mask"].numpy(),
            f"{tag}_allowed": np.array([i for i in range(len(tk)) if i not in ban], np.int64),
            f"{tag}_unit_id": np.array(tk.convert_tokens_to_ids([f"<Un{u}>" for u in range(NUM_UNITS)]), np.int64),
            f"{tag}_marker": np.array(tk.convert_tokens_to_ids("<speech>")),
            f"{tag}_prefix": np.array([1] if bos else [], np.int64),
            f"{tag}_out": gen.numpy(),
            f"{tag}_units": np.concatenate([d.numpy().astype(np.int64) for d in dec] + [np.zeros(0, np.int64)]),
            f"{tag}_units_len": np.array([d.numel() for d in dec]),
        })
        print(tag, "prompt", prompt["input_ids"].tolist(), "generated", gen[:, prompt["input_ids"].shape[1]:].tolist())
    np.savez_compressed(out_path, **out)


if __name__ == "__main__":
    main(os.path.join(ROOT, "tests", "golden", "interleaved_generate_tiny.npz"))
