"""Generate tests/golden/eval_tiny.npz by running the REFERENCE's own `SpeechLM.log_likelihood` in this container.

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_eval_golden.py`); the fixture is committed and is what
tests/test_gpu_eval.py compares `B200SpeechLM.log_likelihood` against.  The reference does not exist on the GPU box, so
nothing at test/bench time imports it.  Shares the reference model builders and helpers of oracle/make_goldens.py.

What is pinned:
  eval_tiny.npz    reference `SpeechLM.log_likelihood` (slamkit/model/speech_lm.py:22-36) and the modelling metric's tie
                   rule (slamkit/metric/modelling_metric.py) on the CPU: the tiny seeded HubertFeatureExtractor of
                   make_goldens.make_hubert_golden inside a `UnitTokeniser`, and the tiny seeded bf16 `UnitLM` of
                   make_goldens.make_loglik_golden (seed 3).  A positive and a negative batch of 4 ragged clips each
                   (pairs 0..3), and one pair whose positive and negative are the same clip, each side a batch of its own
                   (a guaranteed tie).  Stores the clips, the tokens, the bf16 log-likelihoods (mean and sum) and the
                   per-pair results.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_goldens import REF, _reference_unit_lm, _stub_omegaconf, bf16_to_u16  # noqa: E402


def _reference_hubert_fe():
    """The reference's `HubertFeatureExtractor` on the seeded tiny mHuBERT-geometry weights of make_hubert_golden."""
    from sklearn.cluster import KMeans
    from transformers import HubertConfig, HubertModel
    from slamkit.feature_extractor.hubert_feature_extractor import HubertFeatureExtractor
    from oracle.hubert_oracle import OracleHubertConfig, init_hubert_params, hf_state_dict_from_oracle

    ocfg = OracleHubertConfig(conv_dim=64, hidden=128, n_heads=2, ffn=256, n_layers=3, pos_conv_kernel=16,
                              pos_conv_groups=4, n_units=50, layer=3)
    hcfg = HubertConfig(
        hidden_size=ocfg.hidden, num_hidden_layers=ocfg.n_layers, num_attention_heads=ocfg.n_heads,
        intermediate_size=ocfg.ffn, conv_dim=(ocfg.conv_dim,) * 8, conv_stride=ocfg.conv_stride,
        conv_kernel=ocfg.conv_kernel, conv_bias=False, feat_extract_norm="group", do_stable_layer_norm=False,
        num_conv_pos_embeddings=ocfg.pos_conv_kernel, num_conv_pos_embedding_groups=ocfg.pos_conv_groups,
        hidden_dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, feat_proj_dropout=0.0, layerdrop=0.0,
        feat_proj_layer_norm=True, mask_time_prob=0.0, layer_norm_eps=ocfg.ln_eps)
    params = init_hubert_params(ocfg, seed=11)
    model = HubertModel(hcfg).eval()
    model.load_state_dict(hf_state_dict_from_oracle(params, ocfg, model.state_dict()), strict=True)
    km = KMeans(n_clusters=ocfg.n_units, n_init=1)
    km.cluster_centers_ = params["kmeans.centers"].numpy().astype(np.float32)
    km._n_threads = 1
    km.n_features_in_ = ocfg.hidden
    km._n_features_out = ocfg.n_units
    fe = HubertFeatureExtractor.__new__(HubertFeatureExtractor)
    torch.nn.Module.__init__(fe)
    fe.layer, fe.num_units = ocfg.layer, ocfg.n_units
    fe.model, fe.config_model, fe.clustering = model, hcfg, km
    return fe


def make_eval_golden(out_path: str):
    """Writes eval_tiny.npz as described in the module docstring."""
    from oracle.lm_oracle import OracleLMConfig
    from slamkit.model.speech_lm import SpeechLM
    from slamkit.tokeniser.unit_tokeniser import UnitTokeniser

    ocfg = OracleLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256)
    lm, _ = _reference_unit_lm(ocfg, 3)
    lm = lm.to(torch.bfloat16)
    tok = UnitTokeniser(_reference_hubert_fe(), dedup=True, bos_eos_token_id=1, pad_token_id=0, num_units=500)
    slm = SpeechLM(lm, tok, device="cpu")

    g = torch.Generator().manual_seed(21)

    def batch(lens):
        S = max(lens)
        w = torch.zeros(len(lens), S)
        for i, n in enumerate(lens):
            # noise with a slow envelope, so neighbouring frames share units and the dedup has runs to merge
            env = 0.5 + 0.5 * torch.sin(torch.linspace(0, 6.28 * (1 + i), n))
            w[i, :n] = (0.1 * torch.randn(n, generator=g) * env).clamp(-1, 1)
        return w, torch.tensor(lens)

    sides = {"pos": batch([16000, 9600, 12800, 5120]), "neg": batch([11200, 16000, 7040, 13440])}
    tie_wav, tie_len = batch([10880])
    sides["tie_pos"] = (tie_wav, tie_len)
    sides["tie_neg"] = (tie_wav.clone(), tie_len.clone())
    blob = {}
    with torch.inference_mode():
        for name, (w, n) in sides.items():
            blob[f"{name}_wav"], blob[f"{name}_lens"] = w.numpy(), n.numpy()
            blob[f"{name}_tokens"] = tok.tokenise(w, n)["input_ids"].numpy()
            for mean in (True, False):
                ll = slm.log_likelihood(w, n, mean_nll=mean)
                assert ll.dtype == torch.bfloat16, ll.dtype
                blob[f"{name}_ll_{'mean' if mean else 'sum'}_u16"] = bf16_to_u16(ll)

    def pairs(p, q):
        res = torch.zeros_like(p)                  # modelling_metric's tie rule, on the bf16 values
        res[p > q] = 1
        res[p == q] = 0.5
        res[p < q] = 0
        return res.float().numpy()

    u16 = lambda k: torch.from_numpy(blob[k].astype(np.int16)).view(torch.bfloat16)  # noqa: E731
    for form in ("mean", "sum"):
        blob[f"res_{form}"] = pairs(u16(f"pos_ll_{form}_u16"), u16(f"neg_ll_{form}_u16"))
        blob[f"res_tie_{form}"] = pairs(u16(f"tie_pos_ll_{form}_u16"), u16(f"tie_neg_ll_{form}_u16"))
    np.savez_compressed(out_path, **blob)
    print("eval golden ->", out_path, "tokens", {k: v.shape for k, v in blob.items() if k.endswith("_tokens")},
          "res", blob["res_mean"], blob["res_tie_mean"])


if __name__ == "__main__":
    assert os.path.isdir(REF), "the reference is only mounted in the build container"
    _stub_omegaconf()
    sys.path.insert(0, REF)
    make_eval_golden(os.path.join(ROOT, "tests", "golden", "eval_tiny.npz"))
