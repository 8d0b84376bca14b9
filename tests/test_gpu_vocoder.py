"""HiFi-GAN unit vocoder on the GPU (`sk_vocoder_*`, slamkit_b200/vocoder.py) against the reference's own waveforms
(tests/golden/vocoder_tiny.npz, written by oracle/make_vocoder_golden.py) and against an fp64 torch restatement of
the network at the benchmark geometry, plus batch invariance, guard bands, workspace reuse and code validation."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "vocoder_tiny.npz")
REL_L2, MAX_ABS = 1e-4, 2e-4

# the benchmark geometry (tools/vocoder_bench.py): HiFi-GAN V1 widths, 640x upsampling, with a duration predictor
BENCH_CFG = dict(resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3, upsample_rates=[5, 4, 4, 4, 2],
                 upsample_kernel_sizes=[11, 8, 8, 8, 4], upsample_initial_channel=512, model_in_dim=128,
                 num_embeddings=500, embedding_dim=128,
                 dur_predictor_params=dict(encoder_embed_dim=128, var_pred_hidden_dim=128, var_pred_kernel_size=3,
                                           var_pred_dropout=0.5))


def _golden(tag):
    z = np.load(GOLDEN)
    cfg = json.loads(str(z[f"{tag}_config"]))
    sd = {k[len(tag) + 4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"{tag}_sd/")}
    lens = z[f"{tag}_wave_len"]
    offs = np.concatenate([[0], np.cumsum(lens)])
    waves = [z[f"{tag}_wave"][offs[i]:offs[i + 1]] for i in range(len(lens))]
    extra = {k: z[f"{tag}_{k}"] for k in ("log_dur", "dur") if f"{tag}_{k}" in z.files}
    return cfg, sd, torch.from_numpy(z[f"{tag}_codes"]), torch.from_numpy(z[f"{tag}_counts"]), waves, extra


def _close(got, ref, what):
    got, ref = torch.as_tensor(got).double().cpu().reshape(-1), torch.as_tensor(ref).double().cpu().reshape(-1)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if ref.numel() == 0:
        return
    err = got - ref
    rel = float(err.norm() / ref.norm().clamp_min(1e-30))
    mx = float(err.abs().max())
    assert rel <= REL_L2 and mx <= MAX_ABS, f"{what}: rel-L2 {rel:.3e} max-abs {mx:.3e}"


@pytest.fixture(scope="module", params=["a", "b"])
def golden(request):
    from slamkit_b200.vocoder import HifiGanB200Vocoder
    cfg, sd, codes, counts, waves, extra = _golden(request.param)
    voc = HifiGanB200Vocoder(cfg, sd, device="cuda:0", max_rows=16, max_frames=4096)
    return request.param, voc, codes, counts, waves, extra


def test_golden_alone_and_batched(golden):
    tag, voc, codes, counts, waves, extra = golden
    for i in range(codes.shape[0]):
        w = voc.vocode(codes[i, :int(counts[i])])
        _close(w, waves[i], f"{tag} row {i} alone")
    wave, lens = voc.vocode_batch(codes, counts)
    torch.cuda.synchronize()
    for i in range(codes.shape[0]):
        assert int(lens[i]) == len(waves[i])
        _close(wave[i, :int(lens[i])], waves[i], f"{tag} row {i} in the batch")
        assert bool((wave[i, int(lens[i]):] == 0).all())


def test_golden_durations(golden):
    tag, voc, codes, counts, waves, extra = golden
    if "dur" not in extra:
        pytest.skip("geometry without a duration predictor")
    dur, logd, frames, status = voc.durations(codes, counts)
    got_d, got_v = [], []
    for i in range(codes.shape[0]):
        n = int((codes[i, :int(counts[i])] >= 0).sum())
        got_d.append(dur[i, :n].cpu())
        got_v.append(logd[i, :n].cpu())
    got_d, got_v = torch.cat(got_d).numpy(), torch.cat(got_v).numpy()
    ref_v = extra["log_dur"].astype(np.float64)
    assert np.abs(got_v - ref_v).max() < 1e-4
    x = np.exp(ref_v) - 1
    near_half = np.abs(x - np.floor(x) - 0.5) < 1e-4
    assert ((got_d == extra["dur"]) | near_half).all()
    assert int(status.sum()) == 0


# ---- fp64 torch restatement of CodeGenerator (generator.py / resblock.py), TF32 off ---------------------------------
def _restated(cfg, folded, units, dur):
    d = torch.float64
    W = {k: v.to("cuda", d) for k, v in folded.items()}
    x = W["dict.weight"][units].T[None]                                   # [1, E, n]
    x = torch.repeat_interleave(x, dur.to("cuda"), dim=2)
    if cfg.get("multispkr"):
        x = torch.cat([x, W["spkr.weight"][0][None, :, None].expand(1, -1, x.shape[2])], 1)
    if cfg.get("multistyle"):
        x = torch.cat([x, W["style.weight"][0][None, :, None].expand(1, -1, x.shape[2])], 1)
    x = F.conv1d(x, W["conv_pre.weight"], W["conv_pre.bias"], padding=3)
    nk = len(cfg["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        x = F.leaky_relu(x, 0.1)
        x = F.conv_transpose1d(x, W[f"ups.{i}.weight"], W[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        xs = None
        for j, (rk, dl) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            y = x
            p = f"resblocks.{i * nk + j}"
            for a in range(3):
                t = F.conv1d(F.leaky_relu(y, 0.1), W[f"{p}.convs1.{a}.weight"], W[f"{p}.convs1.{a}.bias"],
                             dilation=dl[a], padding=(rk * dl[a] - dl[a]) // 2)
                t = F.conv1d(F.leaky_relu(t, 0.1), W[f"{p}.convs2.{a}.weight"], W[f"{p}.convs2.{a}.bias"],
                             padding=(rk - 1) // 2)
                y = t + y
            xs = y if xs is None else xs + y
        x = xs / nk
    x = F.conv1d(F.leaky_relu(x), W["conv_post.weight"], W["conv_post.bias"], padding=3)
    return torch.tanh(x).reshape(-1)


def _random_state_dict(cfg, seed):
    """Weight-norm pairs of the benchmark geometry with O(1) activations (a textlesslib-layout state dict)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    E, C0 = cfg["embedding_dim"], cfg["upsample_initial_channel"]

    def conv(name, shape, gain):
        v = torch.randn(shape, generator=g)
        sd[name + ".weight_v"] = v
        sd[name + ".weight_g"] = gain * (0.6 + 0.6 * torch.rand((shape[0],) + (1,) * (len(shape) - 1), generator=g))
        sd[name + ".bias"] = 0.05 * torch.randn(shape[1] if name.startswith("ups.") else shape[0], generator=g)

    sd["dict.weight"] = torch.randn(cfg["num_embeddings"], E, generator=g)
    H = cfg["dur_predictor_params"]["var_pred_hidden_dim"]
    for n, s in (("conv1.0", (H, E, 3)), ("conv2.0", (H, H, 3))):
        sd[f"dur_predictor.{n}.weight"] = torch.randn(s, generator=g) / (s[1] * 3) ** 0.5
        sd[f"dur_predictor.{n}.bias"] = 0.05 * torch.randn(H, generator=g)
    for n in ("ln1", "ln2"):
        sd[f"dur_predictor.{n}.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
        sd[f"dur_predictor.{n}.bias"] = 0.1 * torch.randn(H, generator=g)
    sd["dur_predictor.proj.weight"] = 0.5 * torch.randn(1, H, generator=g) / H ** 0.5
    sd["dur_predictor.proj.bias"] = torch.tensor([0.9])
    conv("conv_pre", (C0, cfg["model_in_dim"], 7), 1.0)
    ch = C0
    nk = len(cfg["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        conv(f"ups.{i}", (ch, ch // 2, k), u ** 0.5)
        ch //= 2
        for j, rk in enumerate(cfg["resblock_kernel_sizes"]):
            for a in range(3):
                conv(f"resblocks.{i * nk + j}.convs1.{a}", (ch, ch, rk), 0.5)
                conv(f"resblocks.{i * nk + j}.convs2.{a}", (ch, ch, rk), 0.5)
    conv("conv_post", (1, ch, 7), 1.0)
    return sd


@pytest.fixture(scope="module")
def bench_vocoder():
    from slamkit_b200.vocoder import HifiGanB200Vocoder
    sd = _random_state_dict(BENCH_CFG, seed=5)
    return HifiGanB200Vocoder(BENCH_CFG, sd, device="cuda:0", max_rows=8, max_frames=2048), sd


def test_bench_geometry_vs_fp64_restatement(bench_vocoder):
    from slamkit_b200.vocoder import fold_weight_norm
    voc, sd = bench_vocoder
    g = torch.Generator().manual_seed(7)
    lens = [1, 400, 37, 2, 150, 9, 260, 64]
    codes = torch.full((8, 400), -1, dtype=torch.int64)
    for i, n in enumerate(lens):
        codes[i, :n] = torch.randint(0, 500, (n,), generator=g)
    counts = torch.tensor(lens, dtype=torch.int32)
    dur, _, frames, _ = voc.durations(codes, counts)
    assert int(frames.min()) >= 1
    wave, wl = voc.vocode_batch(codes, counts)
    torch.cuda.synchronize()
    folded = fold_weight_norm(sd)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for i, n in enumerate(lens):
            if i in (1, 6, 3):   # the long rows and one short one: the fp64 restatement is slow at 640x
                ref = _restated(BENCH_CFG, folded, codes[i, :n].cuda(), dur[i, :n].long())
                _close(wave[i, :int(wl[i])], ref, f"row {i} ({n} units)")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_batch_invariance(golden):
    tag, voc, codes, counts, waves, extra = golden
    rows = [codes[i, :int(counts[i])] for i in range(codes.shape[0])]
    alone = [voc.vocode(r).cpu() for r in rows]
    wave, lens = voc.vocode_batch(rows)
    perm = torch.randperm(len(rows), generator=torch.Generator().manual_seed(1)).tolist()
    wave_p, lens_p = voc.vocode_batch([rows[p] for p in perm])
    for i in range(len(rows)):
        assert torch.equal(wave[i, :int(lens[i])].cpu(), alone[i]), f"row {i}: batch != alone"
        assert bool((wave[i, int(lens[i]):] == 0).all())
    for j, p in enumerate(perm):
        assert torch.equal(wave_p[j, :int(lens_p[j])].cpu(), alone[p]), f"row {p}: permuted batch != alone"
        assert bool((wave_p[j, int(lens_p[j]):] == 0).all())


def test_sub_batches_equal_one_batch(golden):
    """A request larger than the workspace is split into sub-batches of whole rows, with identical samples."""
    from slamkit_b200.vocoder import HifiGanB200Vocoder
    tag, voc, codes, counts, waves, extra = golden
    z = _golden(tag)
    small = HifiGanB200Vocoder(z[0], z[1], device="cuda:0", max_rows=3, max_frames=130)
    w1, l1 = voc.vocode_batch(codes, counts)
    w2, l2 = small.vocode_batch(codes, counts)
    assert torch.equal(l1, l2) and torch.equal(w1, w2)


def test_guard_bands_and_workspace_reuse(golden):
    from slamkit_b200 import _lib as L
    from slamkit_b200.vocoder import HifiGanB200Vocoder
    tag, voc, codes, counts, waves, extra = golden
    B = codes.shape[0]
    c, n = codes.cuda(), counts.cuda()
    _, _, frames, _ = voc.durations(c, n)
    fh = frames.cpu().contiguous()
    S = int(fh.max()) * voc.upsampling
    ldw, margin = S + 37, 1024
    buf = torch.full((margin + B * ldw + margin,), 12345.0, device="cuda")
    out = buf[margin:margin + B * ldw]
    L.check(voc.lib.sk_vocoder_run(voc._h, L.ptr(c), c.shape[1], L.ptr(n), B, fh.numpy().ctypes.data_as(C.POINTER(C.c_int32)),
                                   L.ptr(out), C.c_int64(ldw), L.stream_ptr()))
    torch.cuda.synchronize()
    assert bool((buf[:margin] == 12345.0).all()) and bool((buf[margin + B * ldw:] == 12345.0).all())
    ref, lens = voc.vocode_batch(codes, counts)
    o = out.view(B, ldw)
    assert torch.equal(o[:, :S], ref) and bool((o[:, S:] == 0).all())   # the whole pitch is written
    # a long batch then a short one on the same workspace equals the short one on a fresh instance
    voc.vocode_batch(codes[7:10].repeat(4, 1), counts[7:10].repeat(4))
    short, sl = voc.vocode_batch(codes[:3], counts[:3])
    z = _golden(tag)
    fresh = HifiGanB200Vocoder(z[0], z[1], device="cuda:0", max_rows=16, max_frames=4096)
    short2, sl2 = fresh.vocode_batch(codes[:3], counts[:3])
    assert torch.equal(sl, sl2) and torch.equal(short, short2)


def test_code_validation(golden):
    from slamkit_b200._lib import SkError
    tag, voc, codes, counts, waves, extra = golden
    bad = codes[:4].clone()
    bad[2, 0] = voc.geometry["num_embeddings"]
    with pytest.raises(SkError, match="num_embeddings"):
        voc.vocode_batch(bad, counts[:4])
    w = voc.vocode(codes[5, :int(counts[5])])
    _close(w, waves[5], "after an error")
    # negative codes are dropped; a row with nothing left is an empty waveform
    kept = codes[5, :int(counts[5])]
    mixed = torch.stack([torch.cat([torch.tensor([-1, -7]), kept[:4], torch.tensor([-1]), kept[4:]])])
    assert torch.equal(voc.vocode(mixed[0]), w)
    assert voc.vocode(torch.tensor([-1, -1])).numel() == 0


def _textless_checkpoint(tmp_path, num_embeddings=500):
    """Geometry (a) of the fixture with a 500-unit code table, written as a textlesslib checkpoint + JSON config."""
    cfg, sd, *_ = _golden("a")
    cfg = dict(cfg, num_embeddings=num_embeddings)
    sd = dict(sd, **{"dict.weight": torch.randn(num_embeddings, cfg["embedding_dim"],
                                                generator=torch.Generator().manual_seed(3))})
    mp, cp = tmp_path / "voc.pt", tmp_path / "voc.json"
    torch.save({"generator": sd}, str(mp))
    cp.write_text(json.dumps(cfg))
    return str(mp), str(cp)


def test_speech_lm_generate_and_cli_end_to_end(tmp_path):
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from flac_writer import write_flac
    import cli.eval as E
    from cli.extract_features import build_tokeniser
    from slamkit_b200 import metrics as M
    from slamkit_b200.audio_io import load_audio
    from slamkit_b200.config import load_config
    from slamkit_b200.lm import B200UnitLM, LMConfig
    from slamkit_b200.speech_lm import B200SpeechLM
    from slamkit_b200.vocoder import HifiGanB200Vocoder

    ck = tmp_path / "ck"
    lm = B200UnitLM(LMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256),
                    device="cuda:0", max_batch=4, max_seq=128, trainable=False)
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
            "vocoder=vocoder_hubert_25", f"vocoder.model_path={mp}", f"vocoder.config_path={cp}",
            f"metric.data_path={data}/*.flac", "metric.prompt_length=2", f"metric.out_path={out}",
            "metric.generate_kwargs.do_sample=false", "metric.generate_kwargs.max_new_tokens=24"]
    res = E.main(argv)
    gens = res["generate"]
    assert len(gens) == 4
    files = sorted(os.listdir(out))
    assert files == sorted(f"generate_{i}.wav" for i, w in enumerate(gens) if w.numel() > 0)

    # the same prompts, batches and greedy decoding without a vocoder: the continuation units of each row
    cfg = load_config("eval", argv)
    tok = build_tokeniser(cfg, "cuda:0")
    ds = M.PromptDataset(f"{data}/*.flac", prompt_length=2, sample_rate=16000, num_files=5)
    plain = B200SpeechLM(E.load_model(cfg, "cuda:0", max_seq=E.generate_max_seq(cfg, tok, ds)), tok)
    units = M.generate(plain, f"{data}/*.flac", 3, None, 2, sample_rate=16000, num_files=5, num_workers=2,
                       do_sample=False, max_new_tokens=24)["generate"]
    voc = HifiGanB200Vocoder.from_checkpoint(mp, cp, device="cuda:0")
    for i, u in enumerate(units):
        want = voc.vocode(u).cpu()
        assert torch.equal(gens[i].cpu(), want)
        if want.numel():
            assert torch.equal(load_audio(str(out / f"generate_{i}.wav")), want)
            assert bool(torch.isfinite(want).all()) and float(want.abs().max()) > 0
    # the prompt part of each row is build_prompt's units
    for b0 in range(0, len(ds), 3):
        clips = [ds[i][0] for i in range(b0, min(b0 + 3, len(ds)))]
        lens = torch.tensor([len(c) for c in clips])
        wav = torch.zeros(len(clips), int(lens.max()))
        for r, c in enumerate(clips):
            wav[r, :len(c)] = c
        p = tok.build_prompt(wav.cuda(), lens.cuda())
        for r in range(len(clips)):
            ids = p["input_ids"][r][p["attention_mask"][r].bool()]
            assert int(ids[0]) == tok.bos_token_id
            pu = (ids[1:] - tok.offset).cpu()
            assert torch.equal(units[b0 + r][:len(pu)].cpu(), pu)
