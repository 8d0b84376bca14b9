"""GPU tests of speech continuation with interleaved speech-text models: the device prompt (`sk_units_to_prompt`), the
compact head of `allowed_token_ids` (`sk_lm_gather_head`, `sk_lm_prefill_sub`, `sk_lm_decode_step_sub`,
`sk_select_next_sub`) against the full-vocabulary step and the `bad_words_ids` path, and the argument refusals."""
import ctypes as C

import pytest
import torch

from decode_ref import expected_token

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _text_tokeniser(path, bos: bool):
    """A WordLevel text tokenizer saved to `path`, with or without a bos prefix (OPT-style / Qwen2-style)."""
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from transformers import PreTrainedTokenizerFast
    vocab = {"<pad>": 0, "<s>": 1, "</s>": 2, "hello": 3, "world": 4, "<unk>": 5}
    tk = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    if bos:
        tk.post_processor = processors.TemplateProcessing(single="<s> $A", special_tokens=[("<s>", 1)])
    PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>", pad_token="<pad>", bos_token="<s>" if bos else None,
                            eos_token="</s>").save_pretrained(str(path))
    return str(path)


def _interleaved(tmp_path, bos, num_units=500):
    from slamkit_b200.tokeniser import B200InterleavingTokeniser
    return B200InterleavingTokeniser(None, num_units=num_units, load_fe=False,
                                     text_tokeniser_path=_text_tokeniser(tmp_path / f"tk{int(bos)}", bos))


def _host_prompt(it, units):
    """The reference's build_prompt on unit lists: `<Un i>` strings + `<speech>`, the text tokenizer, left padding,
    a trailing eos dropped."""
    tk = it.text_tokeniser
    tk.padding_side = "left"
    enc = tk(["".join(f"<Un{u}>" for u in row) + "<speech>" for row in units], add_special_tokens=True,
             return_tensors="pt", padding=True)
    tk.padding_side = "right"
    ids, mask = enc["input_ids"], enc["attention_mask"]
    if tk.eos_token_id is not None and bool((ids[:, -1] == tk.eos_token_id).any()):
        ids, mask = ids[:, :-1], mask[:, :-1]
    return ids, mask


@pytest.mark.parametrize("bos", [True, False])
def test_prompt_kernel_equals_host_tokeniser(tmp_path, bos):
    it = _interleaved(tmp_path, bos)
    rows = [[], [7], [3, 499, 0, 12, 250], [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
    T = max(len(r) for r in rows)
    units = torch.zeros(len(rows), T, dtype=torch.int32)
    for b, r in enumerate(rows):
        units[b, :len(r)] = torch.tensor(r, dtype=torch.int32)
    counts = torch.tensor([len(r) for r in rows], dtype=torch.int32)
    got = it.prompt_ids(units.to(DEV), counts.to(DEV))
    want_ids, want_mask = _host_prompt(it, rows)
    assert torch.equal(got["input_ids"].cpu(), want_ids)
    assert torch.equal(got["attention_mask"].cpu(), want_mask.long())
    assert it.prompt_layout()["prefix"] == ([1] if bos else [])


def test_decode_units_equals_host_decode(tmp_path):
    it = _interleaved(tmp_path, True)
    tk = it.text_tokeniser
    un = tk.convert_tokens_to_ids(["<Un5>", "<Un0>", "<Un499>", "<speech>", "<text>"])
    row = torch.tensor([0, 1, un[0], 3, un[1], 2, un[3], un[2], un[4], len(tk) + 3, un[0]])
    want = torch.tensor([5, 0, 499, 5])
    assert torch.equal(it.decode_sample(row.to(DEV)).cpu(), want)
    codes = it.decode_units(torch.stack([row, row.flip(0)]).to(DEV)).cpu()
    assert torch.equal(codes[0][codes[0] >= 0], want) and torch.equal(codes[1][codes[1] >= 0], want.flip(0))


# ---------------------------------------------------------------------------------------------- compact head
def _model(arch, V, max_batch=64):
    from slamkit_b200.lm import B200UnitLM
    if arch in ("qwen2", "qwen2-untied"):
        from oracle import lm_oracle as O
        from slamkit_b200.lm import LMConfig
        tie = arch == "qwen2"
        c = O.OracleLMConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256,
                             tie_embeddings=tie)
        cfg = LMConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256,
                       max_positions=256, tie_embeddings=tie)
        p = O.init_params(c, seed=3)
    elif arch == "opt":
        from oracle import opt_oracle as O
        from slamkit_b200.lm import OptLMConfig
        c = O.OracleOptConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
        cfg = OptLMConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
        p = O.init_params(c, seed=3, dtype=torch.bfloat16)
    elif arch == "opt-postln":
        from oracle import opt_postln_oracle as O
        from slamkit_b200.lm import OptPostLnLMConfig
        c = O.OraclePostLnConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
        cfg = OptPostLnLMConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
        p = O.init_params(c, seed=3)
    else:
        from oracle import neox_oracle as O
        from slamkit_b200.lm import NeoxLMConfig
        c = O.OracleNeoxConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
        cfg = NeoxLMConfig(vocab_size=V, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256,
                           rot_dims=c.rot_dims)
        p = O.init_params(c, seed=3)
    m = B200UnitLM(cfg, device=DEV, max_batch=max_batch, max_seq=64, trainable=False)
    m.load_hf_state_dict(p)
    return m


def _prompts(B, T, V, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[0] = T
    ids = torch.zeros(B, T, dtype=torch.long)
    for r in range(B):
        ids[r, :int(lens[r])] = torch.randint(0, V, (int(lens[r]),), generator=g)
    return ids, lens


def _allowed_sets(V):
    g = torch.Generator().manual_seed(11)
    return {
        "units+bos/eos": [1, 2] + list(range(V - 502, V - 2)),
        "scattered": sorted(torch.randperm(V, generator=g)[:300].tolist()),
        "not-multiple-of-64": list(range(5, 5 + 130)),
        "single": [V // 2],
    }


ARCHS = ["qwen2", "qwen2-untied", "opt", "opt-postln", "neox"]


@pytest.mark.parametrize("arch", ARCHS)
def test_compact_logits_bit_identical_to_full_columns(arch):
    """Prefill and three decode steps: the compact logits equal the full step's columns of the allowed ids, bit for
    bit, for B = 1, 7, 64; the compact head's padding rows give zero columns over a NaN-poisoned logits buffer."""
    from slamkit_b200.lm import DecodeSession
    V = 4099
    m = _model(arch, V)
    for B in (1, 7, 64):
        ids, lens = _prompts(B, 9, V, B)
        for name, allowed in _allowed_sets(V).items():
            A = torch.tensor(allowed)
            full = DecodeSession(m, B, 16, 4)
            sub = DecodeSession(m, B, 16, 4, allowed=A)
            sub.logits_buf.fill_(float("nan"))
            lf, ls = full.prefill(ids, lens), sub.prefill(ids, lens)
            Ad = A.to(DEV)
            for s in range(4):
                assert torch.equal(ls.view(torch.int16), lf[:, Ad].contiguous().view(torch.int16)), (arch, B, name, s)
                assert bool((sub.logits_buf[:, A.numel():] == 0).all()), (arch, B, name, s)
                tok = torch.randint(0, V, (B,), generator=torch.Generator().manual_seed(s)).to(DEV)
                pos = (lens + s).to(torch.int32).to(DEV)
                lf, ls = full.step(tok, pos), sub.step(tok, pos)


@pytest.mark.parametrize("V", [4099, 152167])
@pytest.mark.parametrize("eos_inside", [True, False])
def test_greedy_allowed_equals_bad_words(V, eos_inside):
    m = _model("qwen2", V, max_batch=8)
    allowed = [1, 2] + list(range(V - 502, V - 2))
    eos = 2 if eos_inside else 3
    ids, lens = _prompts(5, 12, V, 1)
    T = ids.shape[1]
    left = torch.zeros_like(ids)
    mask = torch.zeros_like(ids)
    for r in range(5):
        n = int(lens[r])
        left[r, T - n:], mask[r, T - n:] = ids[r, :n], 1
    keep = set(allowed)
    bad = [[i] for i in range(V) if i not in keep]
    a = m.generate(left, attention_mask=mask, max_new_tokens=30, eos_token_id=eos, pad_token_id=0,
                   allowed_token_ids=allowed)
    b = m.generate(left, attention_mask=mask, max_new_tokens=30, eos_token_id=eos, pad_token_id=0, bad_words_ids=bad)
    assert torch.equal(a.cpu(), b.cpu())
    assert set(a[:, T:].flatten().tolist()) <= keep | {0}


def test_sampled_num_return_sequences_equals_bad_words():
    V = 4099
    m = _model("neox", V, max_batch=16)
    allowed = list(range(V - 502, V))
    keep = set(allowed)
    bad = [[i] for i in range(V) if i not in keep]
    ids = torch.randint(0, V, (3, 10), generator=torch.Generator().manual_seed(2))
    kw = dict(max_new_tokens=24, do_sample=True, temperature=0.8, top_k=25, top_p=0.9, num_return_sequences=4,
              eos_token_id=None, pad_token_id=0)
    a = m.generate(ids, allowed_token_ids=allowed, generator=torch.Generator().manual_seed(9), **kw)
    b = m.generate(ids, bad_words_ids=bad, generator=torch.Generator().manual_seed(9), **kw)
    assert a.shape == (12, 34) and torch.equal(a.cpu(), b.cpu())


@pytest.mark.parametrize("cfg", [dict(do_sample=False), dict(do_sample=True, temperature=0.8, top_k=25),
                                 dict(do_sample=True, temperature=1.3, top_p=0.7), dict(do_sample=True, top_k=600)])
def test_sampled_compact_selection_equals_reference(cfg):
    """sk_select_next_sub on given compact rows and uniforms picks expected_token's id on the full row with every
    other id banned (rows whose uniform lies within 1e-5 of a CDF boundary are skipped)."""
    L, lib = _lib()
    V, B, max_new = 5000, 32, 4
    g = torch.Generator().manual_seed(4)
    ids = torch.sort(torch.randperm(V, generator=g)[:517]).values
    n = ids.numel()
    ld = (n + 63) // 64 * 64
    logits = (torch.randn(B, n, generator=g) * 3).to(torch.bfloat16)
    logits[:, 7] = logits[:, 9]                                    # a tie
    lg = torch.full((B, ld), float("nan"), dtype=torch.bfloat16)
    lg[:, :n] = logits
    u = torch.rand(B, generator=g)
    sc = L.SkSampling(seed=1, top_p=float(cfg.get("top_p", 1.0)), temperature=float(cfg.get("temperature", 1.0)),
                      do_sample=int(cfg["do_sample"]), top_k=int(cfg.get("top_k", 0)), n_eos=0, pad_token_id=0,
                      max_length=1 << 30)
    z = lambda: torch.zeros(B, dtype=torch.int32, device=DEV)
    pos, fin, ngen = z(), z(), z()
    tokens = torch.zeros(B, dtype=torch.long, device=DEV)
    out = torch.full((B, max_new), -1, dtype=torch.long, device=DEV)
    step = torch.zeros(2, dtype=torch.int32, device=DEV)
    st = L.SkDecodeState(tokens.data_ptr(), pos.data_ptr(), fin.data_ptr(), ngen.data_ptr(), out.data_ptr(),
                         step.data_ptr(), max_new, 0)
    lg_d, ids_d, u_d = lg.to(DEV), ids.to(torch.int32).to(DEV), u.to(DEV)
    L.check(lib.sk_select_next_sub(L.ptr(lg_d), ld, L.ptr(ids_d), n, V, B, C.byref(sc), L.ptr(u_d), C.byref(st),
                                   L.stream_ptr()))
    torch.cuda.synchronize()
    keep = set(ids.tolist())
    banned = [i for i in range(V) if i not in keep]
    checked = 0
    for b in range(B):
        row = torch.full((V,), -30.0)
        row[ids] = logits[b].float()
        want, dist = expected_token(row, cfg["do_sample"], cfg.get("temperature", 1.0), cfg.get("top_k", 0),
                                    cfg.get("top_p", 1.0), banned, float(u[b]))
        if dist < 1e-5:
            continue
        checked += 1
        assert int(tokens[b]) == want and int(out[b, 0]) == want, (b, cfg)
    assert checked >= B // 2


def test_refusals():
    m = _model("qwen2", 4099, max_batch=4)
    ids = torch.randint(0, 4099, (2, 5))
    for bad, word in (([], "empty"), ([3, 3], "duplicate"), ([4099], "allowed_token_ids must be in"),
                      ([-1, 5], "allowed_token_ids must be in")):
        with pytest.raises(ValueError, match=word):
            m.generate(ids, max_new_tokens=3, allowed_token_ids=bad)
    with pytest.raises(ValueError, match="not both"):
        m.generate(ids, max_new_tokens=3, allowed_token_ids=[1, 2], bad_words_ids=[[3]])
    L, lib = _lib()
    head = torch.empty(64, 128, dtype=torch.bfloat16, device=DEV)
    ids_d = torch.tensor([1, 2], dtype=torch.int32, device=DEV)
    assert lib.sk_lm_gather_head(m._h, L.ptr(ids_d), 2, 32, L.ptr(head), L.stream_ptr()) != 0
    assert b"multiple of 64" in lib.sk_last_error()


def test_history_rules_fall_back_to_the_same_result():
    V = 4099
    m = _model("opt", V, max_batch=4)
    allowed = list(range(100, 700))
    keep = set(allowed)
    bad = [[i] for i in range(V) if i not in keep]
    ids = torch.randint(0, V, (3, 8), generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=20, repetition_penalty=1.4, no_repeat_ngram_size=2, eos_token_id=None, pad_token_id=0)
    assert torch.equal(m.generate(ids, allowed_token_ids=allowed, **kw).cpu(), m.generate(ids, bad_words_ids=bad, **kw).cpu())


def test_speech_lm_generate_interleaved_rows_vocode_alone(tmp_path):
    """B200SpeechLM.generate with the interleaved tokeniser (units fed through prompt_ids), a tiny Qwen2 over its
    vocabulary and the stand-in vocoder: each row's waveform equals vocoding that row's units alone."""
    from slamkit_b200.speech_lm import B200SpeechLM
    it = _interleaved(tmp_path, False, num_units=500)
    m = _model("qwen2", len(it), max_batch=8)
    rows = [[4, 8, 15], [16], [23, 42, 4, 8]]
    units = torch.zeros(3, 4, dtype=torch.int32)
    for b, r in enumerate(rows):
        units[b, :len(r)] = torch.tensor(r, dtype=torch.int32)
    counts = torch.tensor([len(r) for r in rows], dtype=torch.int32)

    class FE:
        sample_rate = 16000

        def units_device(self, wav, lens):
            return units.to(DEV), counts.to(DEV)

        def dedup_device(self, ids, nf):
            return ids, None, nf

    it.model = FE()
    tk = it.text_tokeniser
    conts = B200SpeechLM(m, it).generate(torch.zeros(3, 100, device=DEV), max_new_tokens=12, eos_token_id=tk.eos_token_id,
                                         pad_token_id=0)
    prompt = it.prompt_ids(units.to(DEV), counts.to(DEV))
    want = m.generate(prompt["input_ids"], attention_mask=prompt["attention_mask"], max_new_tokens=12,
                      eos_token_id=tk.eos_token_id, pad_token_id=0, allowed_token_ids=it.allowed_ids())
    for b in range(3):
        assert torch.equal(conts[b].cpu(), it.decode_sample(want[b]).cpu())
    from test_gpu_vocoder import _textless_checkpoint          # the vocoder tests' 500-unit stand-in checkpoint
    from slamkit_b200.vocoder import HifiGanB200Vocoder
    voc = HifiGanB200Vocoder.from_checkpoint(*_textless_checkpoint(tmp_path), device=DEV)
    waves = B200SpeechLM(m, it, vocoder=voc).generate(torch.zeros(3, 100, device=DEV), max_new_tokens=12,
                                                      eos_token_id=tk.eos_token_id, pad_token_id=0)
    for b in range(3):
        alone = voc.vocode(conts[b]) if conts[b].numel() else torch.zeros(0, device=DEV)
        assert torch.equal(waves[b], alone)


# ---------------------------------------------------------------------------------------------- against the reference
def _golden():
    import os
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "interleaved_generate_tiny.npz"))


def _golden_tokeniser(tmp_path, tag):
    from oracle.make_interleaved_generate_golden import NUM_UNITS, text_tokeniser
    from slamkit_b200.tokeniser import B200InterleavingTokeniser
    return B200InterleavingTokeniser(None, num_units=NUM_UNITS, load_fe=False,
                                     text_tokeniser_path=text_tokeniser(str(tmp_path / tag), tag == "bos"))


def _golden_units(g):
    n = g["units_len"]
    units = torch.zeros(len(n), max(int(n.max()), 1), dtype=torch.int32)
    at = 0
    for b, k in enumerate(n.tolist()):
        units[b, :k] = torch.from_numpy(g["units"][at:at + k])
        at += k
    return units, torch.from_numpy(n).to(torch.int32)


@pytest.mark.parametrize("tag", ["bos", "nobos"])
def test_prompt_kernel_equals_reference_golden(tmp_path, tag):
    g = _golden()
    it = _golden_tokeniser(tmp_path, tag)
    units, counts = _golden_units(g)
    got = it.prompt_ids(units.to(DEV), counts.to(DEV))
    assert torch.equal(got["input_ids"].cpu(), torch.from_numpy(g[f"{tag}_prompt_ids"]))
    assert torch.equal(got["attention_mask"].cpu(), torch.from_numpy(g[f"{tag}_prompt_mask"]).long())


@pytest.mark.parametrize("tag", ["bos", "nobos"])
def test_golden_model_greedy_equals_hf(tmp_path, tag):
    """The reference's tiny Qwen2 (HF greedy generate with the SPEECH ban list) and ours with allowed_token_ids give
    the same tokens, and decode_sample the same units."""
    from oracle import lm_oracle as O
    from oracle.make_interleaved_generate_golden import MODEL, NEW, SEED, STD
    from slamkit_b200.lm import B200UnitLM, LMConfig
    g = _golden()
    it = _golden_tokeniser(tmp_path, tag)
    V = len(it)
    m = B200UnitLM(LMConfig(vocab_size=V, max_positions=256, **MODEL), device=DEV, max_batch=4, max_seq=32,
                   trainable=False)
    m.load_hf_state_dict(O.init_params(O.OracleLMConfig(vocab_size=V, **MODEL), seed=SEED, std=STD))
    units, counts = _golden_units(g)
    p = it.prompt_ids(units.to(DEV), counts.to(DEV))
    tk = it.text_tokeniser
    out = m.generate(p["input_ids"], attention_mask=p["attention_mask"], max_new_tokens=NEW, eos_token_id=tk.eos_token_id,
                     pad_token_id=0, allowed_token_ids=it.allowed_ids("SPEECH", V))
    assert torch.equal(out.cpu(), torch.from_numpy(g[f"{tag}_out"]))
    n, at = g[f"{tag}_units_len"], 0
    for r in range(out.shape[0]):
        assert it.decode_sample(out[r]).cpu().tolist() == g[f"{tag}_units"][at:at + n[r]].tolist()
        at += n[r]


# ---------------------------------------------------------------------------------------------- HuBERT and the CLI
def _cli_tokeniser(tk_dir):
    import cli.eval as E
    argv = ["model.pretrained_model=/nowhere", "+synthetic_weights=true", "metric=generate", "batch_size=3",
            "tokeniser=interleaved_hubert_25", f"tokeniser.params.text_tokeniser_path={tk_dir}"]
    return E.build_tokeniser(E.load_config("eval", argv), DEV)


def test_prompt_through_synthetic_hubert_equals_host_construction(tmp_path):
    it = _cli_tokeniser(_text_tokeniser(tmp_path / "tk", True))
    g = torch.Generator().manual_seed(4)
    lens = torch.tensor([16000, 4000, 27000])
    wav = torch.zeros(3, 27000)
    for r in range(3):
        wav[r, :int(lens[r])] = 0.1 * torch.randn(int(lens[r]), generator=g)
    got = it.build_prompt(wav.to(DEV), lens.to(DEV))
    rows = [list(r["units"]) for r in it.audio_represent(wav.to(DEV), lens.to(DEV))]
    want_ids, want_mask = _host_prompt(it, rows)
    assert torch.equal(got["input_ids"].cpu(), want_ids)
    assert torch.equal(got["attention_mask"].cpu(), want_mask.long())


def test_cli_generate_interleaved_writes_wavs(tmp_path):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from flac_writer import write_flac
    from test_gpu_vocoder import _textless_checkpoint
    import cli.eval as E
    from slamkit_b200 import metrics as M
    from slamkit_b200.audio_io import load_audio
    from slamkit_b200.lm import B200UnitLM, LMConfig
    from slamkit_b200.speech_lm import B200SpeechLM
    from slamkit_b200.vocoder import HifiGanB200Vocoder

    tk_dir = _text_tokeniser(tmp_path / "tk", True)
    it = _interleaved(tmp_path, True)
    ck = tmp_path / "ck"
    lm = B200UnitLM(LMConfig(vocab_size=len(it), hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256),
                    device=DEV, max_batch=4, max_seq=128, trainable=False)
    lm.init_weights(5, std=0.05)
    lm.save_pretrained(str(ck))
    g = torch.Generator().manual_seed(21)
    data = tmp_path / "prompts"
    data.mkdir()
    for i, n in enumerate((36000, 20000, 52000, 41000)):
        pcm = (0.2 * torch.randn(n, generator=g).clamp(-4, 4) / 4 * 32767).round().long().numpy()[:, None]
        write_flac(str(data / f"p{i}.flac"), pcm)
    mp, cp = _textless_checkpoint(tmp_path)
    out = tmp_path / "gen"
    argv = [f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=3", "num_workers=2", "metric=generate",
            "tokeniser=interleaved_hubert_25", f"tokeniser.params.text_tokeniser_path={tk_dir}",
            "vocoder=vocoder_hubert_25", f"vocoder.model_path={mp}", f"vocoder.config_path={cp}",
            f"metric.data_path={data}/*.flac", "metric.prompt_length=2", f"metric.out_path={out}",
            "metric.generate_kwargs.do_sample=false", "metric.generate_kwargs.max_new_tokens=24"]
    gens = E.main(argv)["generate"]
    assert len(gens) == 4
    assert sorted(os.listdir(out)) == sorted(f"generate_{i}.wav" for i, w in enumerate(gens) if w.numel() > 0)
    # the same prompts and greedy decoding without a vocoder: each file is its row's units vocoded alone
    cfg = E.load_config("eval", argv)
    tok = _cli_tokeniser(tk_dir)
    ds = M.PromptDataset(f"{data}/*.flac", prompt_length=2, sample_rate=16000, num_files=5)
    plain = B200SpeechLM(E.load_model(cfg, DEV, max_seq=E.generate_max_seq(cfg, tok, ds)), tok)
    units = M.generate(plain, f"{data}/*.flac", 3, None, 2, sample_rate=16000, num_files=5, num_workers=2,
                       do_sample=False, max_new_tokens=24)["generate"]
    voc = HifiGanB200Vocoder.from_checkpoint(mp, cp, device=DEV)
    for i, u in enumerate(units):
        want = voc.vocode(u).cpu() if u.numel() else torch.zeros(0)
        assert torch.equal(gens[i].cpu(), want)
        if want.numel():
            assert torch.equal(load_audio(str(out / f"generate_{i}.wav")), want)


# ---------------------------------------------------------------------------------------------- guard bands
def test_guard_bands_and_poisoned_workspace():
    """The compact head and logits are written inside their bounds only (NaN guard rows / columns around them stay as
    they were), and a NaN-poisoned decode workspace gives the same compact logits as a clean one."""
    from slamkit_b200.lm import DecodeSession
    L, lib = _lib()
    V, B = 4099, 7
    m = _model("qwen2", V, max_batch=8)
    A = torch.tensor(sorted(torch.randperm(V, generator=torch.Generator().manual_seed(2))[:100].tolist()))
    ids, lens = _prompts(B, 9, V, 3)
    clean = DecodeSession(m, B, 16, 4, allowed=A)
    n_pad, K = clean.head.shape
    nan16 = torch.tensor(float("nan"), dtype=torch.bfloat16).view(torch.int16)
    # head: 64 guard rows on both sides
    big = torch.full((n_pad + 128, K), float("nan"), dtype=torch.bfloat16, device=DEV)
    ids_d = A.to(torch.int32).to(DEV)
    L.check(lib.sk_lm_gather_head(m._h, L.ptr(ids_d), A.numel(), n_pad, L.ptr(big[64:]), L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(big[64:64 + n_pad], clean.head)
    assert bool((big[:64].view(torch.int16) == nan16).all()) and bool((big[64 + n_pad:].view(torch.int16) == nan16).all())
    # logits: pitch n_pad + 64 and a guard row after the batch
    poisoned = DecodeSession(m, B, 16, 4, allowed=A)
    poisoned.ws.fill_(0xFF)                                      # every bf16 / fp32 slot a NaN
    ld = n_pad + 64
    lg = torch.full((B + 1, ld), float("nan"), dtype=torch.bfloat16, device=DEV)
    assert torch.equal(poisoned.prefill(ids, lens).view(torch.int16), clean.prefill(ids, lens).view(torch.int16))
    for s in range(3):
        tok = torch.randint(0, V, (B,), generator=torch.Generator().manual_seed(s)).to(DEV)
        pos = (lens + s).to(torch.int32).to(DEV)
        want = clean.step(tok, pos).clone()
        assert torch.equal(poisoned.step(tok, pos).view(torch.int16), want.view(torch.int16)), s
        # the same step again into the guarded buffer (it rewrites this token's K/V at pos with the same values)
        L.check(lib.sk_lm_decode_step_sub(m._h, L.ptr(tok), L.ptr(pos), B, L.ptr(poisoned.kv), poisoned.T_cache,
                                          L.ptr(poisoned.head), n_pad, L.ptr(lg), ld, L.ptr(poisoned.ws),
                                          C.c_int64(poisoned.ws.numel()), L.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(lg[:B, :A.numel()].view(torch.int16), want.view(torch.int16)), s
        assert bool((lg[:B, n_pad:].view(torch.int16) == nan16).all()) and bool((lg[B].view(torch.int16) == nan16).all())
