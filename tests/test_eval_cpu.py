"""Host side of cli/eval.py (no GPU): dataset order and pairing, the tie / NaN rule, `//reference` resolution, config
composition and the metric types the CLI refuses."""
import os
import wave

import pytest
import torch

from slamkit_b200 import metrics as M
from slamkit_b200.config import load_config


def _touch_wav(path):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(b"\0\0" * 16)


def _tree(root, files):
    for f in files:
        p = root / f
        p.parent.mkdir(parents=True, exist_ok=True)
        _touch_wav(p)


def test_swuggy_flat_order_and_pairs(tmp_path):
    # integer prefix order, not string order (10 after 9); no two files share a prefix
    _tree(tmp_path, ["10_neg.wav", "2_pos.wav", "9_neg.wav", "1_neg.wav", "0_pos.wav", "3_neg.wav", "readme.txt"])
    (tmp_path / "sub").mkdir()
    _tree(tmp_path / "sub", ["4_x.wav"])                  # not read without subfolder
    ds = M.ModellingMetricDataset(str(tmp_path), sep="_", subfolder=False)
    names = [p.name for p in ds.data]
    assert names == ["0_pos.wav", "1_neg.wav", "2_pos.wav", "3_neg.wav", "9_neg.wav", "10_neg.wav"]
    assert len(ds) == 3
    assert [tuple(os.path.basename(x) for x in ds.pair(i)) for i in range(3)] == [
        ("0_pos.wav", "1_neg.wav"), ("2_pos.wav", "3_neg.wav"), ("9_neg.wav", "10_neg.wav")]


def test_swuggy_subfolders_follow_iterdir(tmp_path):
    _tree(tmp_path, ["a/11_w.wav", "a/3_w.wav", "a/7_w.wav", "a/20_w.wav", "b/5_w.wav", "b/1_w.wav", "c.wav"])
    ds = M.ModellingMetricDataset(str(tmp_path), sep="_", subfolder=True)
    per_dir = {"a": ["3_w.wav", "7_w.wav", "11_w.wav", "20_w.wav"], "b": ["1_w.wav", "5_w.wav"]}
    expect = []
    for d in tmp_path.iterdir():                           # directory order is the filesystem's, as in the reference
        if d.is_dir():
            expect += per_dir[d.name]
    assert [p.name for p in ds.data] == expect
    assert len(ds) == 3


def test_sblimp_plus_separator(tmp_path):
    _tree(tmp_path, ["d/12+b+x.wav", "d/3+a+y.wav", "d/0+a+x.wav", "d/5+b+y.wav"])
    ds = M.ModellingMetricDataset(str(tmp_path), sep="+", subfolder=True)
    assert [p.name for p in ds.data] == ["0+a+x.wav", "3+a+y.wav", "5+b+y.wav", "12+b+x.wav"]
    assert [tuple(os.path.basename(x) for x in ds.pair(i)) for i in range(2)] == [
        ("0+a+x.wav", "3+a+y.wav"), ("5+b+y.wav", "12+b+x.wav")]


def test_salmon_groups_and_empty_group(tmp_path):
    part = "gender_consistency/"
    _tree(tmp_path / part, ["sample_2_b.wav", "sample_0_neg.wav", "sample_2_a.wav", "sample_0_pos.wav",
                            "sample_3_x.wav", "sample_3_w.wav"])           # group 1 is empty and dropped
    ds = M.SalmonDataset(str(tmp_path), part)
    assert len(ds) == 3
    got = [tuple(os.path.basename(x) for x in ds.pair(i)) for i in range(3)]
    assert got == [("sample_0_neg.wav", "sample_0_pos.wav"), ("sample_2_a.wav", "sample_2_b.wav"),
                   ("sample_3_w.wav", "sample_3_x.wav")]
    assert len(M.SALMON_PARTS) == 8


def test_tie_and_nan_rule():
    bf = lambda xs: torch.tensor(xs, dtype=torch.float32).to(torch.bfloat16)  # noqa: E731
    # -2.0039 and -2.0078 both round to bf16 -2.0 (ulp 2^-6 at 2): a tie
    pos = bf([-1.0, -3.0, -2.0039, float("nan"), -1.0, float("nan"), float("-inf"), float("-inf")])
    neg = bf([-2.0, -1.0, -2.0078, -1.0, float("nan"), float("nan"), -5.0, float("-inf")])
    res = M.score_pairs(pos, neg)
    assert res.dtype == torch.bfloat16
    assert res.float().tolist() == [1.0, 0.0, 0.5, 0.0, 0.0, 0.0, 0.0, 0.5]


def test_reference_path_resolution(monkeypatch):
    monkeypatch.delenv("SLAM_REFERENCE_PATH", raising=False)
    assert M.resolve_reference_path("/data/swuggy", None) == "/data/swuggy"
    assert M.resolve_reference_path("//reference/swuggy", "/cfg") == "/cfg/swuggy"
    with pytest.raises(ValueError):
        M.resolve_reference_path("//reference/swuggy", None)
    monkeypatch.setenv("SLAM_REFERENCE_PATH", "/env")
    assert M.resolve_reference_path("//reference/swuggy", "/cfg") == "/env/swuggy"


@pytest.mark.parametrize("metric,mtype,subfolder", [
    ("swuggy_inter", "swuggy", True), ("swuggy_oov", "swuggy", True), ("sblimp", "sblimp", True),
    ("sstorycloze", "storycloze", False), ("tstorycloze", "storycloze", False), ("salmon", "salmon", False)])
def test_eval_config_composes(metric, mtype, subfolder):
    cfg = load_config("eval", [f"metric={metric}"])
    assert cfg.metric.metric_type == mtype
    assert cfg.metric.subfolder is subfolder
    assert cfg.metric.mean_nll is True and cfg.metric.used_token_modality is None and cfg.metric.cross_modal is False
    assert cfg.metric.data_path.startswith("//reference/")
    assert cfg.batch_size == 8 and cfg.num_workers == 8 and cfg.pin_memory is True and cfg.reference_path is None
    assert cfg.vocoder.vocoder_type is None and cfg.model.pretrained_model is None
    if mtype == "salmon":
        assert cfg.metric.parts == ["all"]


def test_eval_config_default_metric_needs_values():
    cfg = load_config("eval", ["metric=default"])
    with pytest.raises(ValueError):
        cfg.metric.metric_type


@pytest.mark.parametrize("mtype", ["generate", "asr_perplexity", "llm_as_judge"])
def test_generative_metrics_raise(mtype):
    import cli.eval as E
    cfg = load_config("eval", [f"metric.metric_type={mtype}"])
    with pytest.raises(NotImplementedError, match="vocoder, Whisper or an external LLM"):
        E.check_metric(cfg)
    with pytest.raises(NotImplementedError):
        E.main([f"metric.metric_type={mtype}", "metric.data_path=/nonexistent"])


def test_cross_modal_and_unknown_metrics_raise():
    import cli.eval as E
    with pytest.raises(NotImplementedError, match="vocoder, Whisper or an external LLM"):
        E.main(["metric=sstorycloze", "metric.cross_modal=true"])
    with pytest.raises(ValueError, match="Unknown metric type"):
        E.main(["metric.metric_type=perplexity"])
    for mt in ("swuggy", "sblimp", "storycloze", "salmon"):
        assert E.check_metric(load_config("eval", [f"metric.metric_type={mt}"])) == mt
