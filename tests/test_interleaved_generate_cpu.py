"""Host side of speech continuation with the interleaved tokeniser: the prompt layout read off the text tokenizer and the
allowed ids of a SPEECH continuation against the reference (tests/golden/interleaved_generate_tiny.npz, written by
oracle/make_interleaved_generate_golden.py), the refusals, the LM rows `metric=generate` sizes the model for, and the
CLI wiring of `metric=generate tokeniser=interleaved_hubert_25` up to the model loader."""
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "interleaved_generate_tiny.npz")


@pytest.mark.parametrize("tag", ["bos", "nobos"])
def test_host_side_matches_reference_golden(tmp_path, tag):
    from oracle.make_interleaved_generate_golden import NUM_UNITS, text_tokeniser
    from slamkit_b200.tokeniser import B200InterleavingTokeniser
    g = np.load(GOLDEN)
    it = B200InterleavingTokeniser(None, num_units=NUM_UNITS, load_fe=False,
                                   text_tokeniser_path=text_tokeniser(str(tmp_path / tag), tag == "bos"))
    lay = it.prompt_layout()
    assert lay["prefix"] == g[f"{tag}_prefix"].tolist()
    assert lay["unit_id"] == g[f"{tag}_unit_id"].tolist()
    assert lay["marker"] == int(g[f"{tag}_marker"])
    assert it.allowed_ids("SPEECH") == g[f"{tag}_allowed"].tolist()
    # ids of the model's vocabulary past the tokenizer's are not in the reference's ban list: allowed as well
    assert it.allowed_ids("SPEECH", vocab_size=len(it) + 3) == g[f"{tag}_allowed"].tolist() + [len(it) + i for i in range(3)]
    # decode_sample of the reference's continuations (prompts included) gives the reference's units
    out, units, n = g[f"{tag}_out"], g[f"{tag}_units"], g[f"{tag}_units_len"]
    for r, start in enumerate(np.concatenate([[0], np.cumsum(n)[:-1]])):
        assert it.decode_sample(torch.from_numpy(out[r])).tolist() == units[start:start + n[r]].tolist()


def _tokeniser(tmp_path, bos: bool, eos_suffix: bool = False):
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from transformers import PreTrainedTokenizerFast
    from slamkit_b200.tokeniser import B200InterleavingTokeniser
    vocab = {"<pad>": 0, "<s>": 1, "</s>": 2, "hello": 3, "world": 4, "<unk>": 5}
    tk = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    single = ("<s> $A" if bos else "$A") + (" </s>" if eos_suffix else "")
    tk.post_processor = processors.TemplateProcessing(single=single, special_tokens=[("<s>", 1), ("</s>", 2)])
    path = tmp_path / f"tk{int(bos)}{int(eos_suffix)}"
    PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>", pad_token="<pad>", bos_token="<s>" if bos else None,
                            eos_token="</s>").save_pretrained(str(path))
    return B200InterleavingTokeniser(None, num_units=500, load_fe=False, text_tokeniser_path=str(path))


@pytest.mark.parametrize("bos,eos_suffix", [(True, False), (False, False), (True, True)])
def test_prompt_layout(tmp_path, bos, eos_suffix):
    it = _tokeniser(tmp_path, bos, eos_suffix)
    tk = it.text_tokeniser
    lay = it.prompt_layout()
    assert lay["prefix"] == ([1] if bos else [])                  # a trailing eos is dropped, as build_prompt drops it
    assert lay["unit_id"] == [tk.convert_tokens_to_ids(f"<Un{u}>") for u in range(500)]
    assert lay["marker"] == tk.convert_tokens_to_ids("<speech>")


def test_allowed_ids_are_the_complement_of_the_speech_ban_list(tmp_path):
    for bos in (True, False):
        it = _tokeniser(tmp_path, bos)
        ban = set(it.get_ignore_tokens("SPEECH"))
        allowed = it.allowed_ids("SPEECH")
        assert allowed == sorted(set(range(len(it))) - ban)
        assert set(it.prompt_layout()["unit_id"]) <= set(allowed)


def test_text_output_and_list_inputs_keep_raising(tmp_path):
    it = _tokeniser(tmp_path, True)
    with pytest.raises(NotImplementedError):
        it.allowed_ids("TEXT")
    with pytest.raises(NotImplementedError):
        it.build_prompt(torch.zeros(1, 10), output_modality="TEXT")
    with pytest.raises(NotImplementedError):
        it.build_prompt([("hello", "TEXT")])
    with pytest.raises(NotImplementedError):
        it.decode_sample(torch.tensor([1, 2]), output_modality="TEXT")


def test_generate_max_seq_counts_prefix_and_marker(tmp_path, monkeypatch):
    import cli.eval as E
    from slamkit_b200 import audio_io
    from slamkit_b200.config import Cfg

    class FE:
        sample_rate = 16000

        @staticmethod
        def frames(n):
            return n // 320

    class DS:
        data = ["a.wav"]

        @staticmethod
        def crop(i):
            return None

    monkeypatch.setattr(audio_io, "audio_info", lambda p: (32000, 16000))
    cfg = Cfg({"metric": Cfg({"generate_kwargs": {"max_new_tokens": 150}})})
    for bos in (True, False):
        it = _tokeniser(tmp_path, bos)
        it.model = FE()
        assert E.generate_max_seq(cfg, it, DS()) == 100 + (1 if bos else 0) + 1 + 150


def test_cli_generate_wiring_reaches_the_model_loader(tmp_path, monkeypatch):
    """`cli/eval.py metric=generate tokeniser=interleaved_hubert_25` with a local text tokenizer: the interleaved
    tokeniser is built around the unit extractor and the model is loaded with the rows the prompts need."""
    import cli.eval as E
    import cli.extract_features as X
    from oracle.make_interleaved_generate_golden import text_tokeniser
    from slamkit_b200 import integration
    from slamkit_b200.audio_io import write_wav_float
    from slamkit_b200.tokeniser import B200InterleavingTokeniser

    class FE:
        sample_rate = 16000

        @staticmethod
        def frames(n):
            return n // 640

    class Unit:
        model = FE()

    data = tmp_path / "data"
    data.mkdir()
    for i, n in enumerate((48000, 64000)):
        write_wav_float(str(data / f"p{i}.wav"), torch.zeros(n), 16000)
    seen = {}

    def load_model(cfg, device, max_seq=256):
        seen["max_seq"], seen["path"] = max_seq, cfg.model.pretrained_model
        raise RuntimeError("reached the model loader")

    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(X, "build_tokeniser", lambda cfg, device, max_batch=None: Unit())
    monkeypatch.setattr(integration, "vocoder_b200_from_cfg", lambda *a, **k: None)
    monkeypatch.setattr(E, "load_model", load_model)
    tk_dir = text_tokeniser(str(tmp_path / "tk"), True)
    argv = ["model.pretrained_model=/nowhere", "metric=generate", "tokeniser=interleaved_hubert_25",
            f"tokeniser.params.text_tokeniser_path={tk_dir}", "vocoder=vocoder_hubert_25", "batch_size=2",
            f"metric.data_path={data}/*.wav", "metric.prompt_length=3", "metric.generate_kwargs.max_new_tokens=20"]
    tok = E.build_tokeniser(E.load_config("eval", argv), "cpu")
    assert isinstance(tok, B200InterleavingTokeniser) and tok.text_tokeniser.name_or_path == tk_dir
    with pytest.raises(RuntimeError, match="reached the model loader"):
        E.main(argv)
    # 3 s prompts at 640 samples per frame: 75 units, + bos + <speech> + 20 new tokens
    assert seen == {"max_seq": 75 + 2 + 20, "path": "/nowhere"}
