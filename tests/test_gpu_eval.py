"""Speech-LM evaluation on the GPU: `sk_seq_loglik` against the reference's bf16 formula in torch, device tokens against
tokenise(), `B200SpeechLM.log_likelihood` against the reference's own SpeechLM (tests/golden/eval_tiny.npz), the
reference's batching in `slamkit_b200.metrics`, and cli/eval.py end to end."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import u16_to_bf16

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TINY = dict(hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256)
QWEN_TEXT = 151665              # Qwen2.5 tokenizer length; + 500 units + <speech>, <text> = 152,167
QWEN_EOS = 151643


def _lm(V, seed=0, max_batch=8, max_seq=128, std=0.1):
    from slamkit_b200.lm import B200UnitLM, LMConfig
    m = B200UnitLM(LMConfig(vocab_size=V, **TINY), device=DEV, max_batch=max_batch, max_seq=max_seq, trainable=False)
    m.init_weights(seed, std=std)
    return m


def _reference_formula(logits, tokens, pad, ignore, mean_nll):
    """UnitLM.log_likelihood + calc_nll of the bf16 reference model, in torch on the same bf16 logits."""
    z = logits.clone()
    if ignore is not None:
        z[:, :, ignore] = float("-inf")
    x = tokens[:, 1:].clone()
    x[x == pad] = -100
    losses = F.cross_entropy(z[:, :-1, :].reshape(-1, z.shape[-1]), x.reshape(-1), reduction="none").view(x.shape)
    return losses, _reduce(losses, x.ne(-100), mean_nll)


def _reduce(losses, mask, mean_nll):
    ll = (losses * mask).sum(dim=-1)
    return -(ll / mask.sum(dim=-1) if mean_nll else ll)


def _bits(t):
    return t.contiguous().view(torch.int16).long()


def _ban_list(kind, V, g):
    if kind is None:
        return None
    if kind == "speech":                           # B200InterleavingTokeniser.get_ignore_tokens("SPEECH") layout
        return [x for x in range(QWEN_TEXT) if x != QWEN_EOS] + [V - 2, V - 1]
    return torch.randperm(V - 2, generator=g)[:400].add(2).tolist()


def _tokens(V, kind, ban, B, T, g):
    """Right-padded rows (pad 0): full, padded at 30, one with no valid target, one with a banned target."""
    if kind == "speech":
        ids = torch.randint(QWEN_TEXT, QWEN_TEXT + 500, (B, T), generator=g)
    else:
        allowed = torch.tensor(sorted(set(range(2, V)) - set(ban or [])))
        ids = allowed[torch.randint(0, len(allowed), (B, T), generator=g)]
    ids[:, 0] = 1
    ids[1, 30:] = 0
    ids[2, 1:] = 0
    if ban:
        ids[3, 10] = ban[len(ban) // 2]
    return ids


@pytest.mark.parametrize("V", [502, 152167])
@pytest.mark.parametrize("kind", [None, "400", "speech"])
def test_seq_loglik_matches_reference_formula(V, kind):
    if kind == "speech" and V != 152167:
        pytest.skip("the SPEECH ban list belongs to the interleaved 152,167-id vocabulary")
    g = torch.Generator().manual_seed(V + (0 if kind is None else len(kind)))
    B, T = 8, 128
    m = _lm(V)
    ban = _ban_list(kind, V, g)
    ids = _tokens(V, kind, ban, B, T, g)
    for mean_nll in (True, False):
        ll, tok = m.sequence_log_likelihood(ids, mean_nll, ban, return_token_nll=True)
        ll2, tok2 = m.sequence_log_likelihood(ids, mean_nll, ban, return_token_nll=True)
        assert ll.dtype == torch.bfloat16 and ll.shape == (B,) and tok.shape == (B, T - 1)
        assert torch.equal(_bits(ll), _bits(ll2)) and torch.equal(tok.view(torch.int32), tok2.view(torch.int32))
        m.forward(ids)
        logits = m.logits_view(B, T)
        ids_d = ids.to(DEV)
        ref_tok, ref_ll = _reference_formula(logits, ids_d, 0, ban, mean_nll)
        # per token: the same bf16 value, or one ulp apart where the fp32 log-sum-exp lands across a rounding boundary
        tb = tok.to(torch.bfloat16)
        assert torch.equal(tb.float(), tok), "token values must be bf16 values"
        fin = torch.isfinite(ref_tok)
        assert torch.equal(fin, torch.isfinite(tb)) and torch.equal(ref_tok[~fin], tb[~fin])
        d = (_bits(tb) - _bits(ref_tok)).abs()[fin]
        assert int(d.max()) <= 1, f"a token differs by {int(d.max())} bf16 ulps"
        assert float((d == 0).float().mean()) >= 0.999, f"{int((d != 0).sum())} of {d.numel()} tokens differ by 1 ulp"
        # per sequence: exactly the reference's reduction applied to the kernel's own token values
        mask = ids_d[:, 1:].ne(0)
        want = _reduce(tb, mask, mean_nll)
        assert torch.equal(torch.isnan(ll), torch.isnan(want))
        ok = ~torch.isnan(want)
        assert torch.equal(_bits(ll)[ok], _bits(want)[ok]), (ll, want)
        # and close to the reference formula on torch's own token values
        assert torch.allclose(ll[ok].float(), ref_ll[ok].float(), rtol=8e-3, atol=0, equal_nan=True)
        # the edge rows: no valid target -> NaN (mean) / 0 (sum); a banned target -> -inf
        assert bool(torch.isnan(ll[2])) if mean_nll else float(ll[2]) == 0.0
        if ban:
            assert float(ll[3]) == float("-inf")
        assert torch.isfinite(ll[[0, 1]].float()).all()


def test_seq_loglik_rejects_bad_arguments():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    x = torch.zeros(4, 16, device=DEV, dtype=torch.bfloat16)
    ids = torch.zeros(2, 2, device=DEV, dtype=torch.long)
    tok = torch.zeros(2, device=DEV)
    ll = torch.zeros(2, device=DEV, dtype=torch.bfloat16)
    s = L.stream_ptr()
    assert lib.sk_seq_loglik(L.ptr(x), 16, 1, L.ptr(ids), 2, 2, 0, None, 1, L.ptr(tok), L.ptr(ll), s) == -1     # V < 2
    assert lib.sk_seq_loglik(L.ptr(x), 12, 10, L.ptr(ids), 2, 2, 0, None, 1, L.ptr(tok), L.ptr(ll), s) == -1    # ldl % 8
    assert lib.sk_seq_loglik(L.ptr(x), 8, 10, L.ptr(ids), 2, 2, 0, None, 1, L.ptr(tok), L.ptr(ll), s) == -1     # ldl < V
    assert lib.sk_seq_loglik(L.ptr(x), 16, 16, L.ptr(ids), 2, 2, 0, None, 1, None, L.ptr(ll), s) == -1         # token_nll
    assert lib.sk_seq_loglik(L.ptr(x), 16, 16, L.ptr(ids), 2, 2, 0, None, 2, L.ptr(tok), L.ptr(ll), s) == -1    # mean_nll
    assert lib.sk_units_to_tokens(L.ptr(ids), L.ptr(ids), 2, 2, 2, 1, 1, 0, L.ptr(ids), 1, s) == -1            # T_out < 2
    m = _lm(502, max_seq=16)
    with pytest.raises(ValueError, match="max_positions"):
        m.sequence_log_likelihood(torch.ones(1, 2049, dtype=torch.long), True)
    with pytest.raises(ValueError, match="right-padding"):
        m.sequence_log_likelihood(torch.ones(1, 4, dtype=torch.long), True,
                                  attention_mask=torch.tensor([[1, 0, 1, 1]]))


# ---------------------------------------------------------------------------------------------- tokens on the device
def _tiny_fe(max_batch=4, max_samples=16000):
    from oracle import hubert_oracle as HO
    from slamkit_b200.feature_extractor import HubertB200Config, HubertB200FeatureExtractor
    o = HO.OracleHubertConfig(conv_dim=64, hidden=128, n_heads=2, ffn=256, n_layers=3, pos_conv_kernel=16,
                              pos_conv_groups=4, n_units=50, layer=3)
    c = HubertB200Config(conv_dim=o.conv_dim, conv_kernel=o.conv_kernel, conv_stride=o.conv_stride, hidden=o.hidden,
                         n_heads=o.n_heads, ffn=o.ffn, layer=o.layer, pos_conv_kernel=o.pos_conv_kernel,
                         pos_conv_groups=o.pos_conv_groups, n_units=o.n_units, ln_eps=o.ln_eps, pad=o.pad)
    return HubertB200FeatureExtractor(c, HO.init_hubert_params(o, seed=11), device=DEV, max_batch=max_batch,
                                      max_samples=max_samples)


def test_units_to_tokens_kernel():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    g = torch.Generator().manual_seed(4)
    units = torch.randint(0, 500, (5, 9), generator=g, dtype=torch.int32)
    counts = torch.tensor([9, 1, 0, 4, 1], dtype=torch.int32)       # full, single unit, empty, ragged
    T_out = 11
    out = torch.full((5, T_out), -7, dtype=torch.long, device=DEV)
    u_d, c_d = units.to(DEV), counts.to(DEV)
    L.check(lib.sk_units_to_tokens(L.ptr(u_d), L.ptr(c_d), 5, 9, 2, 1, 1, 0, L.ptr(out), T_out, L.stream_ptr()))
    for b in range(5):
        n = int(counts[b])
        want = [1] + [int(u) + 2 for u in units[b, :n]] + [1] + [0] * (T_out - n - 2)
        assert out[b].tolist() == want


@pytest.mark.parametrize("dedup", [True, False])
def test_tokenise_device_equals_tokenise(dedup):
    from slamkit_b200.tokeniser import B200UnitTokeniser
    tk = B200UnitTokeniser(_tiny_fe(), dedup=dedup)
    g = torch.Generator().manual_seed(8)
    lens = torch.tensor([16000, 3200, 9000, 640])
    wav = torch.zeros(4, 16000)
    for i, n in enumerate(lens.tolist()):
        wav[i, :n] = 0.1 * torch.randn(n, generator=g)
    wav[3] = 0.0                                   # a silent clip
    for w, n in ((wav, lens), (wav[:1], lens[:1]), (wav[3:], lens[3:]), (wav, None)):
        ids, mask = tk.tokenise_device(w, n)
        ref = tk.tokenise(w, n)
        assert ids.device.type == "cuda"
        assert torch.equal(ids.cpu(), ref["input_ids"]) and torch.equal(mask.cpu(), ref["attention_mask"])
    ids, _ = tk.tokenise_device(wav[3:], lens[3:])
    assert ids.shape[1] == 3, ids                     # the 640-sample clip is a single unit: [BOS, u, EOS]


# ---------------------------------------------------------------------------------------------- against the reference
def _speech_lm():
    from oracle import lm_oracle as O
    from slamkit_b200.lm import B200UnitLM, LMConfig
    from slamkit_b200.speech_lm import B200SpeechLM
    from slamkit_b200.tokeniser import B200UnitTokeniser
    m = B200UnitLM(LMConfig(vocab_size=502, **TINY), device=DEV, max_batch=8, max_seq=64, trainable=False)
    m.load_hf_state_dict(O.init_params(O.OracleLMConfig(vocab_size=502, **TINY), seed=3))
    return B200SpeechLM(m, B200UnitTokeniser(_tiny_fe()))


def test_speech_lm_matches_reference_fixture(golden_dir):
    from slamkit_b200.metrics import score_pairs
    z = np.load(os.path.join(golden_dir, "eval_tiny.npz"))
    slm = _speech_lm()
    got = {}
    for side in ("pos", "neg", "tie_pos", "tie_neg"):
        w, n = torch.from_numpy(z[f"{side}_wav"]), torch.from_numpy(z[f"{side}_lens"])
        ids, _ = slm.tokenise(w, n)
        assert np.array_equal(ids.cpu().numpy(), z[f"{side}_tokens"]), side
        for form, bars in (("mean", (4e-3, 0.02)), ("sum", (4e-3, 0.5))):
            ll = slm.log_likelihood(w, n, mean_nll=form == "mean")
            assert ll.dtype == torch.bfloat16
            ref = u16_to_bf16(z[f"{side}_ll_{form}_u16"])
            assert np.allclose(ll.float().cpu().numpy(), ref.float().numpy(), rtol=bars[0], atol=bars[1]), (side, ll, ref)
            got[(side, form)] = (ll.cpu(), ref, bars)
    for form in ("mean", "sum"):
        pos, rpos, (rtol, atol) = got[("pos", form)]
        neg, rneg, _ = got[("neg", form)]
        res = score_pairs(pos, neg).float().numpy()
        close = np.abs(rpos.float().numpy() - rneg.float().numpy()) <= atol + rtol * np.abs(rneg.float().numpy())
        assert np.array_equal(res[~close], z[f"res_{form}"][~close]), (form, res, z[f"res_{form}"])
        tie = score_pairs(got[("tie_pos", form)][0], got[("tie_neg", form)][0]).float().numpy()
        assert tie.tolist() == [0.5] and z[f"res_tie_{form}"].tolist() == [0.5]


def _write_clips(root, names, g, lo=2400, hi=12000):
    from slamkit_b200.audio_io import write_wav
    for name in names:
        p = root / name
        p.parent.mkdir(parents=True, exist_ok=True)
        n = int(torch.randint(lo, hi, (1,), generator=g))
        write_wav(str(p), 0.2 * torch.randn(n, generator=g).clamp(-4, 4) / 4)


def test_modelling_metric_batching_matches_direct_calls(tmp_path):
    """batch_size 3 over 7 pairs: the positives and the negatives of each batch are tokenised as separate batches."""
    from slamkit_b200 import metrics as M
    from slamkit_b200.audio_io import load_audio
    g = torch.Generator().manual_seed(12)
    _write_clips(tmp_path, [f"{i}_w.wav" for i in range(14)], g)
    ds = M.ModellingMetricDataset(str(tmp_path), sep="_", subfolder=False)
    assert len(ds) == 7
    slm = _speech_lm()
    res = M.pair_scores(slm, ds, None, True, batch_size=3, num_workers=2)
    want = []
    for i in range(0, 7, 3):
        sides = []
        for k in (0, 1):
            wavs = [load_audio(ds.pair(j)[k]) for j in range(i, min(i + 3, 7))]
            lens = torch.tensor([len(w) for w in wavs])
            pad = torch.zeros(len(wavs), int(lens.max()))
            for r, w in enumerate(wavs):
                pad[r, :len(w)] = w
            sides.append(slm.log_likelihood(pad, lens, mean_nll=True))
        want.append(M.score_pairs(*sides))
    want = torch.cat(want)
    assert res.shape == (7,) and torch.equal(res.cpu(), want.cpu())
    assert M.modelling_metric(slm, ds, None, True, batch_size=3, num_workers=2) == pytest.approx(float(want.float().mean()))


def test_cli_eval_end_to_end(tmp_path):
    import cli.eval as E
    from cli.extract_features import build_tokeniser
    from slamkit_b200 import metrics as M
    from slamkit_b200.config import load_config
    from slamkit_b200.speech_lm import B200SpeechLM
    ck = tmp_path / "ck"
    _lm(502, seed=5, std=0.05).save_pretrained(str(ck))
    g = torch.Generator().manual_seed(13)
    sw = tmp_path / "swuggy"
    _write_clips(sw, [f"{d}/{i}_w.wav" for d in ("a", "b") for i in range(4)], g)
    sal = tmp_path / "salmon"
    _write_clips(sal, [f"gender_consistency/sample_{i}_{s}.wav" for i in (0, 2, 3) for s in ("a", "b")], g)
    common = [f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=2", "num_workers=2"]
    runs = [(["metric=swuggy_inter", f"metric.data_path={sw}"], "swuggy"),
            (["metric=salmon", f"metric.data_path={sal}", "metric.parts=[gender_consistency/]"], "salmon")]
    for extra, kind in runs:
        res = E.main(common + extra)
        cfg = load_config("eval", common + extra)
        slm = B200SpeechLM(E.load_model(cfg, DEV), build_tokeniser(cfg, DEV))
        if kind == "swuggy":
            want = M.swuggy(slm, str(sw), None, True, 2, 2, True, True)
            assert set(res) == {"sWUGGY"}
        else:
            want = M.salmon(slm, str(sal), None, True, ["gender_consistency/"], 2, 2)
            assert set(res) == {"gender_consistency/"}
        assert res == want, (res, want)
