"""cli/train.py -- drop-in for the reference entry point (cli/train.py:16-89), driving the sm_90a train step instead of
HF Trainer.

    torchrun --nproc-per-node 8 cli/train.py data.train_path=<tokens.jsonl> data.val_path=<tokens.jsonl> \
        model=slam model.tlm_type=b200 training_args.output_dir=<dir> [+training_args.max_steps=N] [cont_training=true]

Data contract of `init_dataset` (slamkit/data/hf_dataset.py:91-118): tokenise `audio_repr`, chunk to `context_len`, then
either right-pad with 0 and labels = input_ids with pad -> -100 (DataCollatorForLanguageModeling) or, with
`data.packing=true`, flatten the mini-batch into one row with restarting `position_ids` and a -100 label at every
document start (DataCollatorWithFlattening; the reference requires flash_attention_2 for it, cli/train.py:43-45 -- here
the attention kernels are block-diagonal from the same position_ids).  Schedule / clip / AdamW as
config/training_args/default.yaml; evaluation every `eval_steps`, checkpoints `checkpoint-<step>` every `save_steps`
(HF default 500) keeping `save_total_limit`, `cont_training` = HF `resume_from_checkpoint` (true: latest checkpoint
in output_dir; a path: that checkpoint), `run_time` / `train_max_tokens` stoppers (slamkit/trainer/callbacks.py).
`model.config_args.twist_init=false` starts from seeded random weights."""
import glob
import json
import logging
import math
import os
import re
import shutil
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from slamkit_b200.config import load_config, require, to_container  # noqa: E402
from slamkit_b200.tokeniser import B200UnitTokeniser  # noqa: E402

logger = logging.getLogger(__name__)


def parse_run_time(rt) -> int:
    """RunTimeStopperCallback (slamkit/trainer/callbacks.py:15-27): "D-HH:MM:SS" or seconds."""
    if isinstance(rt, int):
        return rt
    days = 0
    if "-" in rt:
        d, rt = rt.split("-")
        days = int(d)
    h, m, s = rt.split(":")
    return days * 86400 + int(h) * 3600 + int(m) * 60 + int(s)


def load_chunks(pattern: str, tok, context_len: int, min_len=None, max_len=None):
    out = []
    for path in sorted(glob.glob(pattern)):
        for line in open(path):
            ids = tok.prepare_sample(json.loads(line))["input_ids"]
            if max_len and len(ids) > max_len:
                continue
            for i in range(0, len(ids), context_len):          # chunk_texts: keep the remainder, no extra specials
                ch = ids[i:i + context_len]
                if min_len and len(ch) < min_len:
                    continue
                out.append(ch)
    return out


def mix_datasets(sets, ratios, stopping_strategy: str = "first_exhausted", seed: int = 0):
    """`datasets.interleave_datasets(sets, probabilities=ratios, seed=0, stopping_strategy=...)` as `init_dataset` calls it
    for list-valued `data.train_path` (slamkit/data/hf_dataset.py:31-54): source indices are drawn 1000 at a time from
    numpy's default_rng(seed); "first_exhausted" stops when any source runs out, "all_exhausted" re-cycles exhausted
    sources until every one has been seen completely."""
    import numpy as np
    rng = np.random.default_rng(seed)
    n = len(sets)
    cur, done, out = [0] * n, [False] * n, []
    if any(len(x) == 0 for x in sets):
        return out
    oversample = stopping_strategy == "all_exhausted"
    while True:
        for src in (int(i) for i in rng.choice(n, size=1000, p=ratios)):
            if (all(done) if oversample else any(done)):
                return out
            out.append(sets[src][cur[src]])
            cur[src] += 1
            if cur[src] >= len(sets[src]):
                done[src] = True
                cur[src] = 0


def collate(chunks, pad_id: int = 0):
    """DataCollatorForLanguageModeling(mlm=False): right-pad, labels = ids with pad -> -100."""
    n = max(len(c) for c in chunks)
    ids = torch.full((len(chunks), n), pad_id, dtype=torch.int64)
    for i, c in enumerate(chunks):
        ids[i, :len(c)] = torch.tensor(c)
    labels = ids.clone()
    labels[ids == pad_id] = -100
    return {"input_ids": ids, "labels": labels}


def collate_flattened(chunks, separator_id: int = -100):
    """DataCollatorWithFlattening (HF:data/data_collator.py:1364-1440): the whole mini-batch as ONE row of
    sum(len) tokens, labels = separator_id at each document start then the document's own ids, position_ids restarting
    at 0 per document (what marks the document boundaries for the attention kernels)."""
    ids, labels, pos = [], [], []
    for c in chunks:
        ids += list(c)
        labels += [separator_id] + list(c[1:])
        pos += list(range(len(c)))
    t = lambda x: torch.tensor([x], dtype=torch.int64)
    return {"input_ids": t(ids), "labels": t(labels), "position_ids": t(pos)}


def build_tokeniser(cfg):
    t, p = cfg.tokeniser, cfg.tokeniser.params
    if t.tokeniser_type == "unit":
        return B200UnitTokeniser(None, dedup=p.dedup, bos_eos_token_id=p.get("bos_eos_token_id", 1), pad_token_id=p.pad_token_id,
                                 num_units=p.get("num_units") or t.feature_extractor.num_units, load_fe=False)
    if t.tokeniser_type == "interleave":
        from slamkit_b200.tokeniser import B200InterleavingTokeniser
        if p.text_tokeniser_path != cfg.model.config_args.base_model_name:                 # reference cli/train.py:18-23
            logger.warning(f"Text tokeniser {p.text_tokeniser_path}, doesn't match model changing it to: "
                           f"{cfg.model.config_args.base_model_name}")
            p.text_tokeniser_path = cfg.model.config_args.base_model_name
        return B200InterleavingTokeniser(None, dedup=p.dedup, pad_token_id=p.pad_token_id,
                                         num_units=p.get("num_units") or t.feature_extractor.num_units, load_fe=False,
                                         text_tokeniser_path=p.text_tokeniser_path, interleave_method=p.get("interleave_method", "random"),
                                         interleave_span=p.get("interleave_span"), interleave_prob=p.get("interleave_prob"))
    raise ValueError(f"Unknown tokeniser type: {t.tokeniser_type}")                         # audio_tokeniser.py:121


def build_model(cfg, device: str, max_batch: int, max_seq: int):
    """tlm_factory (slamkit/model/token_lm.py:30-43).  The base model's config / weights come from the HF hub (or a
    local directory); when they are unreachable (offline box) the run fails -- unless training from scratch was asked for
    (`twist_init=false`), in which case the decoder shape is taken from `model.shape.*` (default: Qwen2.5-0.5B) and said so."""
    from slamkit_b200.lm import B200UnitLM, LMConfig
    if cfg.model.tlm_type not in ("twist", "gslm", "b200"):
        raise ValueError(f"Unknown slm type: {cfg.model.tlm_type}")                        # token_lm.py:43
    args = cfg.model.config_args
    try:
        from slamkit_b200.integration import tlm_b200_from_cfg
        return tlm_b200_from_cfg(to_container(cfg.model), device=device, max_batch=max_batch, max_seq=max_seq,
                                 autocast_bf16=cfg.training_args.get("bf16"))
    except OSError as e:       # HF hub / local path lookup failures are OSErrors; anything else is a real error
        if args.get("twist_init", True):
            raise RuntimeError(f"base model '{args.base_model_name}' is unreachable and twist_init=true needs its weights "
                               "(set model.config_args.twist_init=false to train from scratch)") from e
        lm_cfg = LMConfig(vocab_size=args.vocab_size, rope_theta=float(args.get("rope_theta", 10000)))
        for k in ("hidden", "n_layers", "n_heads", "n_kv_heads", "ffn"):
            if cfg.model.get("shape", {}).get(k) is not None:
                setattr(lm_cfg, k, cfg.model.shape[k])
        lm_cfg.max_positions = max(lm_cfg.max_positions, int(cfg.model.context_len))
        logger.warning(f"base model config '{args.base_model_name}' unreachable ({type(e).__name__}): twist_init=false, building a "
                       f"seeded random-init Qwen2 decoder of shape {lm_cfg}")
        return B200UnitLM(lm_cfg, device=device, max_batch=max_batch, max_seq=max_seq, seed=0)


# ---- checkpoints (HF Trainer layout: output_dir/checkpoint-<global_step>) ------------------------------------------------
_CKPT_RE = re.compile(r"^checkpoint-(\d+)$")


def list_checkpoints(output_dir: str):
    if not os.path.isdir(output_dir):
        return []
    found = [(int(m.group(1)), os.path.join(output_dir, d)) for d in os.listdir(output_dir) if (m := _CKPT_RE.match(d))]
    return [p for _, p in sorted(found)]


def save_checkpoint(output_dir: str, step: int, model, tok, trainer, extra: dict, save_total_limit=None) -> str:
    path = os.path.join(output_dir, f"checkpoint-{step}")
    os.makedirs(path, exist_ok=True)
    model.save_pretrained(path, base_model_name=extra.get("base_model_name", "Qwen/Qwen2.5-0.5B"))
    tok.save_pretrained(path)
    sd = trainer.state_dict()
    torch.save({"exp_avg": sd["exp_avg"].cpu(), "exp_avg_sq": sd["exp_avg_sq"].cpu(), "opt_step_count": sd["opt_step_count"]},
               os.path.join(path, "optimizer.pt"))
    state = {"global_step": step, "num_input_tokens_seen": sd["num_input_tokens_seen"], **{k: v for k, v in extra.items() if k != "base_model_name"}}
    json.dump(state, open(os.path.join(path, "trainer_state.json"), "w"))
    if save_total_limit:                                            # HF `_rotate_checkpoints`: drop the oldest
        ck = list_checkpoints(output_dir)
        for old in ck[:max(0, len(ck) - int(save_total_limit))]:
            shutil.rmtree(old, ignore_errors=True)
    return path


def main(argv=None):
    argv = list(argv if argv is not None else sys.argv[1:])
    config_name = "train"
    for flag in ("--config-name", "-cn"):                              # hydra's flag: e.g. --config-name train_inter_scale
        if flag in argv:
            i = argv.index(flag)
            config_name = argv[i + 1]
            del argv[i:i + 2]
    cfg = load_config(config_name, argv)
    require(cfg, "data.train_path", "data.val_path")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    ta = cfg.training_args
    # Update num_epochs based on stopping tokens (reference cli/train.py:25-29)
    if cfg.get("train_max_tokens") is not None and (cfg.get("ds_token_size") or 0) > 0:
        ta.num_train_epochs = (cfg.train_max_tokens / cfg.ds_token_size) * 1.01
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    tok = build_tokeniser(cfg)
    if cfg.model.config_args.vocab_size == -1:
        cfg.model.config_args.vocab_size = len(tok)
    ctx = cfg.model.context_len
    d = cfg.data
    if isinstance(d.train_path, list):                                   # config/data/pretrain_multi_ds.yaml
        assert len(d.train_path) == len(d.train_ratios), "Number of train paths should match number of train ratios"
        vps = [d.val_path] if isinstance(d.val_path, str) else list(d.val_path)
        assert len(d.train_path) >= len(vps), "Number of train paths should be more or equal than number of val paths"
        reps = d.get("repetitions") or [1] * len(d.train_path)
        sets = [load_chunks(tp, tok, ctx, d.get("chunk_units_min_length"), d.get("sample_units_max_length")) * int(r)
                for tp, r in zip(d.train_path, reps)]
        train = mix_datasets(sets, list(d.train_ratios), d.get("stopping_strategy", "first_exhausted"))
        val = [c for vp in vps if vp is not None for c in load_chunks(vp, tok, ctx)]
    else:
        train = load_chunks(d.train_path, tok, ctx, d.get("chunk_units_min_length"), d.get("sample_units_max_length"))
        val = load_chunks(d.val_path, tok, ctx)
    if not train:
        raise ValueError(f"no training chunks found under {d.train_path}")
    packing = bool(cfg.data.get("packing", False))
    bs, ga = ta.per_device_train_batch_size, ta.gradient_accumulation_steps
    ebs = ta.get("per_device_eval_batch_size", bs)
    make_batch = collate_flattened if packing else (lambda ch: collate(ch, tok.pad_token_id))
    # a packed mini-batch is one row of up to bs * context_len tokens
    max_b, max_t = (1, max(bs, ebs) * ctx) if packing else (max(bs, ebs), ctx)

    from slamkit_b200.trainer import B200Trainer
    model = build_model(cfg, f"cuda:{local_rank}", max_b, max_t)

    steps_per_epoch = max(1, math.ceil(len(train) / (bs * ga * world)))
    total_steps = ta.get("max_steps") or int(math.ceil(steps_per_epoch * ta.num_train_epochs))
    warmup = ta.get("warmup_steps", 0)
    if warmup > 0 and ta.get("warmup_ratio", 0.0) > 0 and total_steps * ta.warmup_ratio > warmup:
        warmup = int(math.ceil(total_steps * ta.warmup_ratio))                             # cli/train.py:48-54
    elif warmup == 0 and ta.get("warmup_ratio", 0.0) > 0:
        warmup = int(math.ceil(total_steps * ta.warmup_ratio))
    min_lr = (ta.get("lr_scheduler_kwargs") or {}).get("min_lr", 0.0)
    trainer = B200Trainer(model, lr=ta.learning_rate, min_lr=min_lr, warmup_steps=warmup, total_steps=total_steps,
                          max_grad_norm=ta.max_grad_norm, weight_decay=ta.get("weight_decay", 0.0), grad_accum=ga,
                          min_token_id_count=ta.get("min_token_id_count"), max_token_id_count=ta.get("max_token_id_count"))
    budget = parse_run_time(cfg.run_time) if cfg.get("run_time") is not None else None
    max_tokens = cfg.get("train_max_tokens")
    g = torch.Generator().manual_seed(ta.get("seed", 42))
    order = torch.randperm(len(train), generator=g).tolist()
    step, cursor, log = 0, 0, []

    # ---- resume (HF `trainer.train(resume_from_checkpoint=cfg.cont_training)`, reference cli/train.py:89) ----
    resume = cfg.get("cont_training", False)
    if resume:
        ck = resume if isinstance(resume, str) else (list_checkpoints(ta.output_dir) or [None])[-1]
        if ck is None:
            raise ValueError(f"No valid checkpoint found in output directory ({ta.output_dir})")   # HF's message
        from safetensors.torch import load_file
        model.load_hf_state_dict(load_file(os.path.join(ck, "model.safetensors")))
        opt = torch.load(os.path.join(ck, "optimizer.pt"), map_location="cpu")
        st = json.load(open(os.path.join(ck, "trainer_state.json")))
        trainer.load_state_dict({"step_idx": st["global_step"], "num_input_tokens_seen": st["num_input_tokens_seen"],
                                 "opt_step_count": opt["opt_step_count"], "exp_avg": opt["exp_avg"], "exp_avg_sq": opt["exp_avg_sq"]})
        step, cursor, log = st["global_step"], st["cursor"], st.get("log_history", [])
        logger.info(f"resumed from {ck} at step {step}")

    def evaluate():
        ev_nll, ev_n = torch.zeros((), device=model.device, dtype=torch.float64), torch.zeros((), device=model.device, dtype=torch.float64)
        for i in range(rank * ebs, len(val), ebs * world):          # whole eval batches round-robin over ranks
            b = make_batch(val[i:i + ebs])
            out = model.forward(b["input_ids"], labels=b["labels"], position_ids=b.get("position_ids"))
            ev_nll += out.stats[2].double()
            ev_n += out.stats[1].double()
        if world > 1:
            dist.all_reduce(ev_nll)
            dist.all_reduce(ev_n)
        return float(ev_nll / ev_n.clamp(min=1))                    # token-weighted mean NLL over the validation set

    def extra_state():
        return {"cursor": cursor, "log_history": log, "base_model_name": cfg.model.config_args.base_model_name}

    t0 = time.time()
    logging_steps = ta.get("logging_steps", 500)                     # HF TrainingArguments defaults
    eval_steps = ta.get("eval_steps") if ta.get("eval_strategy", "no") == "steps" else None
    save_steps = ta.get("save_steps", 500) if ta.get("save_strategy", "steps") == "steps" else None
    stop = False
    while step < total_steps and not stop:
        micro = []
        for _ in range(ga):
            idx = [order[(cursor + rank * bs + i) % len(order)] for i in range(bs)]
            cursor += bs * world
            micro.append(make_batch([train[i] for i in idx]))
        trainer.train_step(micro)
        step += 1
        if budget is not None and time.time() - t0 > budget:
            stop = True                                             # RunTimeStopperCallback: stop, evaluate, save
        if max_tokens is not None and trainer.num_input_tokens_seen >= max_tokens:
            stop = True                                             # MaxTokensStopperCallback
        last = stop or step == total_steps
        if step % logging_steps == 0 or last:
            rec = {"step": step, "loss": trainer.reduced_loss(), "num_input_tokens_seen": trainer.num_input_tokens_seen,
                   "elapsed_s": time.time() - t0}
            log.append(rec)
            if rank == 0:
                print(json.dumps(rec), flush=True)
        if eval_steps and (step % eval_steps == 0 or stop) and val:
            rec = {"step": step, "eval_loss": evaluate()}
            log.append(rec)
            if rank == 0:
                print(json.dumps(rec), flush=True)
        if save_steps and (step % save_steps == 0 or stop) and rank == 0:
            save_checkpoint(ta.output_dir, step, model, tok, trainer, extra_state(), ta.get("save_total_limit"))
    eval_loss = evaluate() if val else float("nan")
    if rank == 0:
        os.makedirs(ta.output_dir, exist_ok=True)
        model.save_pretrained(ta.output_dir, base_model_name=cfg.model.config_args.base_model_name)   # HF UnitLM layout
        tok.save_pretrained(ta.output_dir)
        json.dump({"log_history": log, "eval_loss": eval_loss, "global_step": step,
                   "num_input_tokens_seen": trainer.num_input_tokens_seen}, open(os.path.join(ta.output_dir, "trainer_state.json"), "w"))
        print(json.dumps({"eval_loss": eval_loss, "steps": step}), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return log


if __name__ == "__main__":
    main()
