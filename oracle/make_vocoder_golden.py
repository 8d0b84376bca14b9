"""Generate tests/golden/vocoder_tiny.npz by running the REFERENCE's own `CodeHiFiGANVocoder` in this container.

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_vocoder_golden.py`); the fixture is committed and is
what tests/test_gpu_vocoder.py compares `HifiGanB200Vocoder` against.  The reference does not exist on the GPU box, so
nothing at test/bench time imports it.

What is pinned, for two seeded tiny geometries:
  a  single speaker with a duration predictor: rates [5, 4, 2], kernels [11, 8, 4], ResBlocks 3/7/11 x dilations
     1/3/5; the predictor's `proj` is biased so that durations of 1 to 5 occur;
  b  multispkr + multistyle, no duration predictor: rates [4, 2], kernels [8, 4], ResBlocks 3/5 with dilations 1/3/5
     and 1/2/4.
For each: the generator's JSON config, its raw state dict (weight_g / weight_v pairs, as a textlesslib checkpoint
stores them), 12 ragged code sequences (one of length 1, ones with -1 entries, one with only -1 entries, long ones), and
each sequence's waveform from `CodeHiFiGANVocoder.forward(code, dur_prediction=...)` vocoded ALONE on the CPU in fp32
(speaker 0, style 0, as `HiFiGANVocoder.vocode` calls it).  For (a) also the predictor's value before exp / round and
the durations of each kept unit.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_goldens import REF, _stub_omegaconf  # noqa: E402

GEOMETRIES = {
    "a": dict(resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3, upsample_rates=[5, 4, 2],
              upsample_kernel_sizes=[11, 8, 4], upsample_initial_channel=32, model_in_dim=32, num_embeddings=50,
              embedding_dim=32, sampling_rate=16000,
              dur_predictor_params=dict(encoder_embed_dim=32, var_pred_hidden_dim=32, var_pred_kernel_size=3,
                                        var_pred_dropout=0.5)),
    "b": dict(resblock_kernel_sizes=[3, 5], resblock_dilation_sizes=[[1, 3, 5], [1, 2, 4]], upsample_rates=[4, 2],
              upsample_kernel_sizes=[8, 4], upsample_initial_channel=32, model_in_dim=48, num_embeddings=40,
              embedding_dim=16, multispkr=True, num_speakers=4, multistyle=True, num_styles=3, sampling_rate=16000),
}


def randomise(model, seed: int, dur_bias: float = 0.9):
    """Weight-norm magnitudes and directions that keep activations O(1) through the stack (the reference's own init,
    N(0, 0.01), vocodes near-silence), random biases and embeddings, and a duration predictor biased to 1..5 frames."""
    g = torch.Generator().manual_seed(seed)
    sd = model.state_dict()
    for k, t in sd.items():
        if k.endswith("weight_v"):
            t.copy_(torch.randn(t.shape, generator=g))
        elif k.endswith("weight_g"):
            stage_up = 1.0
            if k.startswith("ups."):
                stage_up = float(model.ups[int(k.split(".")[1])].stride[0]) ** 0.5
            lo, hi = (0.3, 0.7) if k.startswith("resblocks.") else (0.6, 1.2)
            t.copy_((lo + (hi - lo) * torch.rand(t.shape, generator=g)) * stage_up)
        elif k.endswith("bias"):
            t.copy_(0.05 * torch.randn(t.shape, generator=g))
        elif k in ("dict.weight", "spkr.weight", "style.weight"):
            t.copy_(torch.randn(t.shape, generator=g))
        elif k.startswith("dur_predictor.") and "ln" not in k:
            t.copy_(torch.randn(t.shape, generator=g) / t.shape[-1] ** 0.5 * (2.0 if "conv" in k else 1.0))
        elif k.startswith("dur_predictor.ln"):
            t.copy_((1.0 if k.endswith("weight") else 0.0) + 0.1 * torch.randn(t.shape, generator=g))
    if model.dur_predictor is not None:
        sd["dur_predictor.proj.weight"].mul_(0.5)
        sd["dur_predictor.proj.bias"].fill_(dur_bias)
    model.load_state_dict(sd)


def sequences(num_emb: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    seqs = []
    for n in (1, 2, 3, 5, 8, 13, 21, 34, 48, 64):
        seqs.append(torch.randint(0, num_emb, (n,), generator=g))
    s = torch.randint(0, num_emb, (17,), generator=g)
    s[[0, 4, 5, 16]] = -1
    seqs.append(s)
    seqs.append(torch.full((3,), -1, dtype=torch.int64))
    return seqs


def make_vocoder_golden(out_path: str):
    _stub_omegaconf()
    tmp = tempfile.mkdtemp()
    os.environ["TEXTLESS_CHECKPOINT_ROOT"] = tmp
    from slamkit.vocoder.hifigan.generator import CodeGenerator
    from slamkit.vocoder.hifigan.vocoder import CodeHiFiGANVocoder

    out = {}
    for gi, (tag, cfg) in enumerate(GEOMETRIES.items()):
        torch.manual_seed(100 + gi)
        gen = CodeGenerator(cfg)
        randomise(gen, seed=200 + gi)
        sd = {k: v.clone() for k, v in gen.state_dict().items()}
        mp, cp = os.path.join(tmp, f"{tag}.pt"), os.path.join(tmp, f"{tag}.json")
        torch.save({"generator": sd}, mp)
        with open(cp, "w") as f:
            json.dump(cfg, f)
        voc = CodeHiFiGANVocoder(mp, cp).eval()
        has_dur = voc.model.dur_predictor is not None
        seqs = sequences(cfg["num_embeddings"], seed=300 + gi)
        waves, logd, durs = [], [], []
        with torch.no_grad():
            for s in seqs:
                kept = s[s >= 0]
                if kept.numel() == 0:
                    waves.append(np.zeros(0, np.float32))
                    continue
                y = voc(s.view(1, -1), dur_prediction=has_dur)
                waves.append(y.reshape(-1).numpy().astype(np.float32))
                if has_dur:
                    x = voc.model.dict(kept.view(1, -1))
                    v = voc.model.dur_predictor(x)
                    logd.append(v.reshape(-1).numpy())
                    durs.append(torch.clamp(torch.round(torch.exp(v) - 1).long(), min=1).reshape(-1).numpy())
        n = max(len(s) for s in seqs)
        codes = np.full((len(seqs), n), -1, np.int64)
        for i, s in enumerate(seqs):
            codes[i, :len(s)] = s.numpy()
        out[f"{tag}_config"] = np.array(json.dumps(cfg))
        for k, v in sd.items():
            out[f"{tag}_sd/{k}"] = v.numpy()
        out[f"{tag}_codes"] = codes
        out[f"{tag}_counts"] = np.array([len(s) for s in seqs], np.int32)
        out[f"{tag}_wave"] = np.concatenate(waves)
        out[f"{tag}_wave_len"] = np.array([len(w) for w in waves], np.int64)
        if has_dur:
            out[f"{tag}_log_dur"] = np.concatenate(logd).astype(np.float32)
            out[f"{tag}_dur"] = np.concatenate(durs).astype(np.int32)
        print(tag, "wave lengths", out[f"{tag}_wave_len"].tolist(), "rms", float(np.sqrt((out[f"{tag}_wave"] ** 2).mean())))
        if has_dur:
            print(tag, "durations", np.bincount(out[f"{tag}_dur"]).tolist())
    np.savez_compressed(out_path, **out)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, REF)
    make_vocoder_golden(os.path.join(ROOT, "tests", "golden", "vocoder_tiny.npz"))
