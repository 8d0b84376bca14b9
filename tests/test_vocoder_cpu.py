"""Host side of the unit vocoder and `metric=generate` (no GPU needed): config parsing and refusals, the weight-norm
fold, checkpoint resolution, the float WAV writer, the prompt dataset, metric selection and the prompt layout."""
import json
import os

import numpy as np
import pytest
import torch

from slamkit_b200.config import load_config

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "vocoder_tiny.npz")


def _cfg(tag="a"):
    return json.loads(str(np.load(GOLDEN)[f"{tag}_config"]))


def test_parse_config_and_refusals():
    from slamkit_b200.vocoder import parse_config
    a, b = parse_config(_cfg("a")), parse_config(_cfg("b"))
    assert a["dur_predictor"] and a["dur_hidden"] == 32 and a["upsample_rates"] == [5, 4, 2]
    assert not b["dur_predictor"] and b["multispkr"] and b["multistyle"] and b["model_in_dim"] == 48
    assert a["sampling_rate"] == 16000
    bad = [
        (dict(f0=True), "f0"),
        (dict(embedder_params={"x": 1}), "embedder_params"),
        (dict(upsample_kernel_sizes=[10, 8, 4]), "even"),
        (dict(dur_predictor_params=dict(_cfg("a")["dur_predictor_params"], var_pred_kernel_size=5)), "padding=1"),
        (dict(model_in_dim=64), "model_in_dim"),
    ]
    for change, msg in bad:
        with pytest.raises(ValueError, match=msg):
            parse_config(dict(_cfg("a"), **change))


def test_weight_norm_fold_matches_torch():
    from slamkit_b200.vocoder import fold_weight_norm
    z = np.load(GOLDEN)
    sd = {k[len("a_sd/"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("a_sd/")}
    folded = fold_weight_norm(sd)
    assert not any(k.endswith(("weight_g", "weight_v")) for k in folded)
    for base in ("conv_pre", "ups.0", "ups.2", "resblocks.4.convs1.1", "conv_post"):
        g, v = sd[base + ".weight_g"], sd[base + ".weight_v"]
        want = torch._weight_norm(v.double(), g.double(), 0).float()
        assert torch.allclose(folded[base + ".weight"], want, rtol=1e-6, atol=1e-7), base
    assert sd["ups.0.weight_g"].shape == (32, 1, 1)     # ConvTranspose1d: dim 0 is the input channel


def test_checkpoint_resolution(tmp_path, monkeypatch):
    from slamkit_b200.integration import vocoder_b200_from_cfg, vocoder_checkpoint_paths
    monkeypatch.setenv("TEXTLESS_CHECKPOINT_ROOT", str(tmp_path))
    m, c = vocoder_checkpoint_paths("mhubert-base-25hz", "kmeans", 500)
    assert m == str(tmp_path / "hifigan_lj_mhubert_base_25hz.pt")
    assert c == str(tmp_path / "hifigan_lj_mhubert_base_25hz_config.json")
    m, _ = vocoder_checkpoint_paths("hubert-base-ls960-layer-9", "kmeans", 500)
    assert m.endswith("hifigan_expresso_lj_vctk_hubert_base_ls960_L9_km500_generator.pt")
    cfg = load_config("eval", ["vocoder=vocoder_hubert_25"])
    with pytest.raises(FileNotFoundError, match="hifigan_lj_mhubert_base_25hz.pt"):
        vocoder_b200_from_cfg(cfg.vocoder)
    with pytest.raises(FileNotFoundError, match="nope.pt"):
        vocoder_b200_from_cfg(dict(cfg.vocoder, model_path=str(tmp_path / "nope.pt"), config_path=str(tmp_path / "c")))
    assert vocoder_b200_from_cfg(load_config("eval", []).vocoder) is None
    with pytest.raises(ValueError, match="Unknown vocoder type"):
        vocoder_b200_from_cfg({"vocoder_type": "wavenet"})
    assert load_config("eval", ["vocoder=default"]).vocoder.dense_model_name == "hubert-base-ls960-layer-9"


def test_float_wav_round_trip(tmp_path):
    from scipy.io import wavfile
    from slamkit_b200.audio_io import audio_info, load_audio, write_wav_float
    x = torch.randn(4321, generator=torch.Generator().manual_seed(0)) * 0.3
    p = str(tmp_path / "x.wav")
    write_wav_float(p, x, 16000)
    sr, y = wavfile.read(p)
    assert sr == 16000 and y.dtype == np.float32 and np.array_equal(y, x.numpy())
    assert torch.equal(load_audio(p), x)
    assert audio_info(p) == (4321, 16000)


def test_prompt_dataset(tmp_path):
    from slamkit_b200 import metrics as M
    from slamkit_b200.audio_io import write_wav
    g = torch.Generator().manual_seed(1)
    (tmp_path / "sub").mkdir()
    lens = {"a.wav": 8000, "b.wav": 40000, "sub/c.wav": 30000, "sub/d.wav": 3000}
    for name, n in lens.items():
        write_wav(str(tmp_path / name), 0.1 * torch.randn(n, generator=g))
    pat = str(tmp_path / "**" / "*.wav")
    from glob import glob, iglob
    assert M.PromptDataset(pat).data == glob(pat, recursive=True)
    assert len(M.PromptDataset(pat).data) == 4
    ds = M.PromptDataset(pat, min_file_length=1.0)
    assert sorted(os.path.basename(p) for p in ds.data) == ["b.wav", "c.wav"]
    first = list(iglob(pat, recursive=True))
    ds = M.PromptDataset(pat, num_files=2, min_file_length=0.3)
    assert ds.data == [p for p in first if lens[os.path.relpath(p, tmp_path)] >= 4800][:2]
    ds = M.PromptDataset(pat, prompt_length=1.5)
    for i, p in enumerate(ds.data):
        a, n = ds[i]
        assert n == min(lens[os.path.relpath(p, tmp_path)], 24000) and a.shape == (n,)
    # alignment cut: the word end nearest to prompt_length
    json.dump({"aligned_text": [["w", 0.0, 0.4], ["x", 0.4, 1.3], ["y", 1.3, 1.9]]}, open(tmp_path / "b.json", "w"))
    ds = M.PromptDataset(str(tmp_path / "b.wav"), prompt_length=1.5, use_alignment=True)
    assert ds[0][1] == int(float(torch.tensor(1.3)) * 16000)   # float32 end times, as the reference reads them
    assert M.get_cut_location([("a", 0, 1.0), ("b", 1.0, 2.0)], 1.5) == 1.0
    af = tmp_path / "align"
    af.mkdir()
    json.dump({"aligned_text": [["w", 0.0, 1.8]]}, open(af / "b.json", "w"))
    ds = M.PromptDataset(str(tmp_path / "b.wav"), prompt_length=1.5, use_alignment=True, alignment_folder=str(af))
    assert ds[0][1] == int(float(torch.tensor(1.8)) * 16000)


def test_check_metric_with_and_without_vocoder():
    import cli.eval as E
    assert E.check_metric(load_config("eval", ["metric=generate", "vocoder=vocoder_hubert_25"])) == "generate"
    assert E.check_metric(load_config("eval", ["metric=generate", "vocoder=vocoder_hubert_25",
                                               "vocoder.vocoder_type=hifigan_b200"])) == "generate"
    with pytest.raises(NotImplementedError, match="vocoder, Whisper or an external LLM"):
        E.check_metric(load_config("eval", ["metric=generate"]))
    for mt in ("asr_perplexity", "llm_as_judge"):
        with pytest.raises(NotImplementedError):
            E.check_metric(load_config("eval", [f"metric.metric_type={mt}", "vocoder=vocoder_hubert_25"]))
    with pytest.raises(NotImplementedError):
        E.check_metric(load_config("eval", ["metric=generate", "vocoder=vocoder_hubert_25", "metric.cross_modal=true"]))
    cfg = load_config("eval", ["metric=generate"])
    assert cfg.metric.prompt_length == 3 and cfg.metric.num_files == 5 and cfg.metric.out_path == "generated"
    assert cfg.metric.generate_kwargs.max_new_tokens == 150 and cfg.vocoder.vocoder_type is None


def test_prompt_ids_host():
    from slamkit_b200.tokeniser import B200UnitTokeniser
    t = B200UnitTokeniser(speech_tokeniser=None, load_fe=False)
    units = torch.tensor([[5, 7, 9, 0], [3, 0, 0, 0], [1, 2, 3, 4]], dtype=torch.int32)
    counts = torch.tensor([3, 1, 4])
    p = t.prompt_ids(units, counts)
    # the reference: left-padded `<S> units <S>` through the tokenizer, then the last column (EOS) dropped
    ref = t.string_tokenise(["<Un5><Un7><Un9>", "<Un3>", "<Un1><Un2><Un3><Un4>"])["input_ids"]
    n = max(len(r) for r in ref)
    want = torch.tensor([[0] * (n - len(r)) + r for r in ref])[:, :-1]
    mask = torch.tensor([[0] * (n - len(r)) + [1] * len(r) for r in ref])[:, :-1]
    assert torch.equal(p["input_ids"], want) and torch.equal(p["attention_mask"], mask)
    assert torch.equal(t.decode_sample(p["input_ids"][0]), torch.tensor([5, 7, 9]))
