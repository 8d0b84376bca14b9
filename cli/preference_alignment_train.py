"""cli/preference_alignment_train.py -- drop-in for the reference entry point (cli/preference_alignment_train.py:18-69):
DPO of a unit LM on prompt / chosen / rejected unit strings, on the sm_90a train path.

    torchrun --nproc-per-node N cli/preference_alignment_train.py data.train_path=<pairs.jsonl> data.val_path=<pairs.jsonl> \
        model.pretrained_model=<dir written by cli/train.py> training_args.output_dir=<dir> [+training_args.max_steps=K]

Data: `init_preference_optimization_dataset` (slamkit/data/hf_dataset.py:138-148): jsonl rows, optional repetition filter
on `prompt_text + " " + chosen_text` (auto-BLEU-n of the transcript, calculation_utils.py:30-47), every column but
prompt / chosen / rejected dropped.  Step: `SLAMDPOTrainer` = trl `DPOTrainer` with the BOS/EOS rule of `tokenize_row`,
sigmoid loss, beta 0.1, frozen copy of the initial policy as reference (slamkit_b200/dpo.py).  trl and nltk are not in
the image: truncation uses trl's documented defaults (max_prompt_length 512, max_length 1024 unless given in
training_args), and the repetition filter splits words with a regular expression instead of nltk's Treebank tokeniser
(identical n-grams on plain lower-case transcripts; parity otherwise unpinned)."""
import glob
import json
import logging
import math
import os
import re
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from cli.train import parse_run_time  # noqa: E402
from slamkit_b200.config import load_config, require  # noqa: E402
from slamkit_b200.dpo import collate_pairs, tokenize_row  # noqa: E402
from slamkit_b200.tokeniser import B200UnitTokeniser  # noqa: E402

logger = logging.getLogger(__name__)
_WORD = re.compile(r"\w+|[^\w\s]")


def auto_bleu(text: str, n: int) -> float:
    """calc_auto_bleu (slamkit/utils/calculation_utils.py:30-47): share of word n-grams that occur more than once."""
    tokens = _WORD.findall(text)
    ngrams = [" ".join(tokens[i:i + n]) for i in range(len(tokens) - n + 1)]
    if not ngrams:
        return 0.0
    counts = {}
    for g in ngrams:
        counts[g] = counts.get(g, 0) + 1
    return sum(1 for g in ngrams if counts[g] > 1) / len(ngrams)


def load_pairs(pattern: str, repetition_filter: bool, auto_bleu_n: int, max_auto_bleu: float):
    rows = []
    for path in sorted(glob.glob(pattern)):
        for line in open(path):
            x = json.loads(line)
            if repetition_filter and auto_bleu(x["prompt_text"] + " " + x["chosen_text"], auto_bleu_n) >= max_auto_bleu:
                continue
            rows.append({k: x[k] for k in ("prompt", "chosen", "rejected")})
    return rows


def tokenize_pairs(rows, tok, max_prompt_length, max_length):
    """trl DPOTrainer preprocessing: tokenize_row, then prompt+completion cut to max_length (completion side)."""
    out = []
    for r in rows:
        t = tokenize_row(r, tok, max_prompt_length, None)
        if max_length is not None:
            room = max(1, max_length - len(t["prompt_input_ids"]))
            t["chosen_input_ids"] = t["chosen_input_ids"][:room]
            t["rejected_input_ids"] = t["rejected_input_ids"][:room]
        out.append(t)
    return out


def main(argv=None):
    cfg = load_config("preference_alignment_train", argv if argv is not None else sys.argv[1:])
    require(cfg, "data.train_path")
    if cfg.tokeniser.tokeniser_type == "interleave":
        raise ValueError("Interleave tokeniser not supported for Preference Alignment yet")     # reference :20-21
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    ta, p = cfg.training_args, cfg.tokeniser.params
    tok = B200UnitTokeniser(None, dedup=p.dedup, bos_eos_token_id=p.get("bos_eos_token_id", 1), pad_token_id=p.pad_token_id,
                            num_units=p.get("num_units") or cfg.tokeniser.feature_extractor.num_units, load_fe=False)
    if cfg.model.config_args.vocab_size == -1:
        cfg.model.config_args.vocab_size = len(tok)
    d = cfg.data
    rows = load_pairs(d.train_path, d.get("repetition_filter", False), d.get("auto_bleu_n", 2), d.get("max_auto_bleu", 0.3))
    max_len = ta.get("max_length", 1024)
    pairs = tokenize_pairs(rows, tok, ta.get("max_prompt_length", 512), max_len)
    if not pairs:
        raise ValueError(f"no preference pairs left from {d.train_path}")

    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from cli.train import build_model
    from slamkit_b200.dpo import B200DPOTrainer
    from slamkit_b200.lm import B200UnitLM, cosine_with_min_lr
    bs, ga = ta.per_device_train_batch_size, ta.get("gradient_accumulation_steps", 1)
    dev = f"cuda:{local_rank}"

    def build():
        if cfg.model.get("pretrained_model"):
            return B200UnitLM.from_pretrained(cfg.model.pretrained_model, device=dev, max_batch=2 * bs, max_seq=max_len)
        return build_model(cfg, dev, 2 * bs, max_len)     # same rules as cli/train.py: no silent random-init fallback
    policy, reference = build(), build()          # trl: the reference is a frozen copy of the initial policy
    steps_per_epoch = max(1, math.ceil(len(pairs) / (bs * ga * world)))
    total = ta.get("max_steps") or int(math.ceil(steps_per_epoch * ta.num_train_epochs))
    warmup = ta.get("warmup_steps", 0)
    min_lr = (ta.get("lr_scheduler_kwargs") or {}).get("min_lr", 0.0)
    # data parallel as trl under accelerate DDP (reference cli/preference_alignment_train.py:56-65): every rank takes its
    # own pairs, gradients are summed over ranks with the 1/world factor folded into the per-sequence weights
    trainer = B200DPOTrainer(policy, reference, beta=ta.get("beta", 0.1), lr=ta.learning_rate,
                             max_grad_norm=ta.max_grad_norm, weight_decay=ta.get("weight_decay", 0.0), grad_accum=ga)
    budget = parse_run_time(cfg.run_time) if cfg.get("run_time") is not None else None
    order = torch.randperm(len(pairs), generator=torch.Generator().manual_seed(ta.get("seed", 42))).tolist()
    t0, cursor, log = time.time(), 0, []
    for step in range(1, total + 1):
        mids, mlabs = [], []
        for _ in range(ga):
            batch = [pairs[order[(cursor + rank * bs + i) % len(order)]] for i in range(bs)]
            cursor += bs * world
            ids, labels = collate_pairs(batch, tok.pad_token_id)
            mids.append(ids)
            mlabs.append(labels)
        lr = cosine_with_min_lr(step - 1, base_lr=ta.learning_rate, min_lr=min_lr, warmup_steps=warmup, total_steps=total)
        out = trainer.step(mids, mlabs, lr=lr)
        if step % ta.get("logging_steps", 10) == 0 or step == total:
            vals = {k: v.float().mean() for k, v in out.items() if torch.is_tensor(v)}
            if world > 1:                                     # report the mean over ranks, as trl's gathered metrics
                for v in vals.values():
                    dist.all_reduce(v)
                    v /= world
            rec = {"step": step, "elapsed_s": time.time() - t0, **{k: float(v) for k, v in vals.items()}}
            log.append(rec)
            if rank == 0:
                print(json.dumps(rec), flush=True)
        if budget is not None and time.time() - t0 > budget:
            break
    if rank == 0:
        os.makedirs(ta.output_dir, exist_ok=True)
        policy.save_pretrained(ta.output_dir, base_model_name=cfg.model.config_args.base_model_name)
        tok.save_pretrained(ta.output_dir)
        json.dump({"log": log}, open(os.path.join(ta.output_dir, "trainer_state.json"), "w"))
    if world > 1:
        dist.destroy_process_group()
    return log


if __name__ == "__main__":
    main()
