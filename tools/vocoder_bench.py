"""HiFi-GAN unit vocoder (`sk_vocoder_*`) on the benchmark geometry: embedding 128, 512 initial channels, rates
[5, 4, 4, 4, 2] with kernels [11, 8, 8, 8, 4] (640x: 16 kHz from 25 Hz units), ResBlocks 3/7/11 x dilations 1/3/5 and a
duration predictor, seeded random weights.  The real mhubert-base-25hz vocoder config is not reachable offline; this is
HiFi-GAN V1's widths at that upsampling, a stated stand-in.

Reports, in one run, with the card name and power limit:
  1. the vocoder alone at B = 1, 8, 64 rows of 300 frames (12 s; the predictor is biased to 1 frame per unit, so the
     row length is fixed): ms per `vocode_batch` call (CUDA events, the call's one host read included), audio-seconds
     per second and achieved FLOP/s from the layer shapes -- fp32-equivalent, and as tensor-core work (x3 for the split
     bf16 products) against the 989 TFLOP/s dense-bf16 data-sheet figure;
  2. the same network in torch fp32 (cuDNN, TF32 off) on the same device and batches;
  3. `metric=generate` end to end on synthetic 3 s prompts with the cfg-2 LM (Qwen2.5-0.5B body, 502 units, random
     weights; temperature 0.8, top-k 25, 150 new tokens): prompts per second, split into HuBERT units + prompt ids, LM
     generate and the vocoder.
Prints one line per measurement and a final JSON line.

    python tools/vocoder_bench.py [--batches 1,8,64] [--frames 300] [--e2e-batch 64]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

BF16_TFLOPS, FP32_TFLOPS = 989.0, 67.0     # H100 SXM data sheet, dense (ceilings, not measured rates)
CFG = dict(resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3, upsample_rates=[5, 4, 4, 4, 2],
           upsample_kernel_sizes=[11, 8, 8, 8, 4], upsample_initial_channel=512, model_in_dim=128, num_embeddings=500,
           embedding_dim=128, sampling_rate=16000,
           dur_predictor_params=dict(encoder_embed_dim=128, var_pred_hidden_dim=128, var_pred_kernel_size=3,
                                     var_pred_dropout=0.5))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:   # noqa: BLE001
        q = f"unavailable ({e})"
    return name, q


def state_dict(seed=0):
    """textlesslib-layout weights with O(1) activations; the duration predictor says 1 frame for every unit."""
    g = torch.Generator().manual_seed(seed)
    sd, E, C0 = {}, CFG["embedding_dim"], CFG["upsample_initial_channel"]

    def conv(name, shape, gain):
        sd[name + ".weight_v"] = torch.randn(shape, generator=g)
        sd[name + ".weight_g"] = gain * (0.6 + 0.6 * torch.rand((shape[0],) + (1,) * (len(shape) - 1), generator=g))
        sd[name + ".bias"] = 0.05 * torch.randn(shape[1] if name.startswith("ups.") else shape[0], generator=g)

    sd["dict.weight"] = torch.randn(CFG["num_embeddings"], E, generator=g)
    H = CFG["dur_predictor_params"]["var_pred_hidden_dim"]
    for n, s in (("conv1.0", (H, E, 3)), ("conv2.0", (H, H, 3))):
        sd[f"dur_predictor.{n}.weight"] = torch.randn(s, generator=g) / (s[1] * 3) ** 0.5
        sd[f"dur_predictor.{n}.bias"] = torch.zeros(H)
    for n in ("ln1", "ln2"):
        sd[f"dur_predictor.{n}.weight"], sd[f"dur_predictor.{n}.bias"] = torch.ones(H), torch.zeros(H)
    sd["dur_predictor.proj.weight"] = torch.zeros(1, H)
    sd["dur_predictor.proj.bias"] = torch.tensor([0.6931])      # exp(v) - 1 = 1 frame
    conv("conv_pre", (C0, CFG["model_in_dim"], 7), 1.0)
    ch, nk = C0, len(CFG["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(CFG["upsample_rates"], CFG["upsample_kernel_sizes"])):
        conv(f"ups.{i}", (ch, ch // 2, k), u ** 0.5)
        ch //= 2
        for j, rk in enumerate(CFG["resblock_kernel_sizes"]):
            for a in range(3):
                conv(f"resblocks.{i * nk + j}.convs1.{a}", (ch, ch, rk), 0.5)
                conv(f"resblocks.{i * nk + j}.convs2.{a}", (ch, ch, rk), 0.5)
    conv("conv_post", (1, ch, 7), 1.0)
    return sd


def flops(frames):
    """(fp32-equivalent FLOP of the network on `frames` unit frames, of which tensor-core convolutions)."""
    C0, E = CFG["upsample_initial_channel"], CFG["model_in_dim"]
    T, ch = frames, C0
    tc = 2 * C0 * E * 7 * T
    for u, k in zip(CFG["upsample_rates"], CFG["upsample_kernel_sizes"]):
        tc += 2 * ch * (ch // 2) * k * T          # transposed: every input meets every tap once
        T, ch = T * u, ch // 2
        tc += 2 * ch * ch * sum(CFG["resblock_kernel_sizes"]) * 2 * 3 * T
    return tc + 2 * ch * 7 * T, tc


def torch_fp32(folded, units, dur):
    W = folded
    x = W["dict.weight"][units].transpose(1, 2)
    x = torch.repeat_interleave(x, dur, dim=2)
    x = F.conv1d(x, W["conv_pre.weight"], W["conv_pre.bias"], padding=3)
    nk = len(CFG["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(CFG["upsample_rates"], CFG["upsample_kernel_sizes"])):
        x = F.conv_transpose1d(F.leaky_relu(x, 0.1), W[f"ups.{i}.weight"], W[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        xs = None
        for j, (rk, dl) in enumerate(zip(CFG["resblock_kernel_sizes"], CFG["resblock_dilation_sizes"])):
            y, p = x, f"resblocks.{i * nk + j}"
            for a in range(3):
                t = F.conv1d(F.leaky_relu(y, 0.1), W[f"{p}.convs1.{a}.weight"], W[f"{p}.convs1.{a}.bias"], dilation=dl[a],
                             padding=(rk * dl[a] - dl[a]) // 2)
                y = F.conv1d(F.leaky_relu(t, 0.1), W[f"{p}.convs2.{a}.weight"], W[f"{p}.convs2.{a}.bias"],
                             padding=(rk - 1) // 2) + y
            xs = y if xs is None else xs + y
        x = xs / nk
    return torch.tanh(F.conv1d(F.leaky_relu(x), W["conv_post.weight"], W["conv_post.bias"], padding=3)).squeeze(1)


def timed(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--e2e-batch", type=int, default=64)
    ap.add_argument("--skip-e2e", action="store_true")
    a = ap.parse_args()
    from slamkit_b200.vocoder import HifiGanB200Vocoder, fold_weight_norm
    if not torch.cuda.is_available():
        raise SystemExit("vocoder_bench needs a CUDA device")
    name, limits = card()
    print(f"card: {name}; power limit, max SM clock: {limits}")
    batches = [int(x) for x in a.batches.split(",")]
    sd = state_dict()
    Bmax, Fr = max(batches), a.frames
    voc = HifiGanB200Vocoder(CFG, sd, device="cuda:0", max_rows=Bmax, max_frames=Bmax * Fr)
    folded = {k: v.cuda() for k, v in fold_weight_norm(sd).items()}
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    res = {"card": name, "power_limit_and_max_sm_clock": limits, "frames_per_row": Fr, "vocoder": [], "torch_fp32": []}
    g = torch.Generator().manual_seed(1)
    for B in batches:
        codes = torch.randint(0, 500, (B, Fr), generator=g).cuda()
        wave, lens = voc.vocode_batch(codes)
        assert int(lens.min()) == int(lens.max()) == Fr * 640, "the benchmark needs 1 frame per unit"
        n = max(3, 192 // B)
        ms = timed(lambda: voc.vocode_batch(codes), n)
        fl, tc = flops(Fr)
        fl, tc = fl * B, tc * B
        sec = B * Fr * 640 / 16000
        r = dict(B=B, ms=ms, audio_s_per_s=sec / (ms / 1e3), tflops_fp32_equiv=fl / ms / 1e9,
                 tflops_tensor_core=3 * tc / ms / 1e9, share_of_bf16_peak=3 * tc / ms / 1e9 / BF16_TFLOPS)
        res["vocoder"].append(r)
        print(f"vocoder B={B} x {Fr} frames ({sec:.0f} s of audio): {ms:.2f} ms per batch, {r['audio_s_per_s']:.0f} audio-s/s, "
              f"{r['tflops_fp32_equiv']:.1f} TFLOP/s fp32-equivalent, {r['tflops_tensor_core']:.1f} TFLOP/s tensor-core work "
              f"(x3 split) = {100 * r['share_of_bf16_peak']:.1f} % of the {BF16_TFLOPS:.0f} TFLOP/s dense-bf16 data sheet "
              "(compute-bound: the activations are read once per layer)")
        units = codes
        dur = torch.ones(Fr, dtype=torch.long, device="cuda")
        with torch.inference_mode():
            y = torch_fp32(folded, units, dur)
            d = (y - wave).double()
            rel = float(d.norm() / y.double().norm())
            tms = timed(lambda: torch_fp32(folded, units, dur), max(2, n // 2))
        t = dict(B=B, ms=tms, audio_s_per_s=sec / (tms / 1e3), tflops_fp32=fl / tms / 1e9, rel_l2_vs_vocoder=rel)
        res["torch_fp32"].append(t)
        print(f"torch fp32 (cuDNN, TF32 off) B={B}: {tms:.2f} ms per batch, {t['audio_s_per_s']:.0f} audio-s/s, "
              f"{t['tflops_fp32']:.1f} TFLOP/s of the {FP32_TFLOPS:.0f} fp32 data sheet; vocoder vs torch rel-L2 {rel:.2e}; "
              f"speed-up {tms / ms:.2f}x")
        del wave, y
        torch.cuda.empty_cache()
    if not a.skip_e2e:
        res["generate_e2e"] = e2e(voc, a.e2e_batch)
    print(json.dumps(res))


def e2e(voc, B):
    """metric=generate's device work for one batch of B synthetic 3 s prompts, timed stage by stage."""
    from slamkit_b200.feature_extractor import HubertB200Config, HubertB200FeatureExtractor, random_params
    from slamkit_b200.lm import B200UnitLM, LMConfig
    from slamkit_b200.tokeniser import B200UnitTokeniser
    hc = HubertB200Config(layer=11, n_units=500)
    fe = HubertB200FeatureExtractor(hc, random_params(hc, seed=0), device="cuda:0", max_batch=B, max_samples=48000)
    tok = B200UnitTokeniser(fe)
    lm = B200UnitLM(LMConfig(vocab_size=502), device="cuda:0", max_batch=B, max_seq=256, trainable=False, seed=0)
    g = torch.Generator().manual_seed(2)
    wav = (0.1 * torch.randn(B, 48000, generator=g)).cuda()
    lens = torch.full((B,), 48000, device="cuda")
    kw = dict(do_sample=True, temperature=0.8, top_k=25, max_new_tokens=150, generator=torch.Generator().manual_seed(0))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    out = {}
    for rep in range(3):                  # the first pass warms up (graph capture, cuDNN, allocator)
        torch.cuda.synchronize()
        ev[0].record()
        p = tok.build_prompt(wav, lens)
        ev[1].record()
        conts = lm.generate(p["input_ids"], attention_mask=p["attention_mask"], **kw)
        decoded = [tok.decode_sample(c) for c in conts]
        ev[2].record()
        w, wl = voc.vocode_batch(decoded)
        ev[3].record()
        torch.cuda.synchronize()
        hub, gen, vo = (ev[i].elapsed_time(ev[i + 1]) for i in range(3))
        if rep:
            out = dict(B=B, hubert_ms=hub, generate_ms=gen, vocoder_ms=vo, prompts_per_s=B / ((hub + gen + vo) / 1e3),
                       mean_units_per_row=sum(len(d) for d in decoded) / B,
                       audio_s=float(wl.sum()) / 16000)
    print(f"metric=generate end to end, B={B} synthetic 3 s prompts, cfg-2 LM, 150 new tokens: "
          f"{out['prompts_per_s']:.1f} prompts/s; HuBERT + prompt {out['hubert_ms']:.1f} ms, LM generate "
          f"{out['generate_ms']:.1f} ms, vocoder {out['vocoder_ms']:.1f} ms ({out['mean_units_per_row']:.0f} units per row, "
          f"{out['audio_s']:.0f} s of audio)")
    return out


if __name__ == "__main__":
    main()
