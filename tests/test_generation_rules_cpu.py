"""CPU tests of the history-dependent generation rules of slamkit_b200/generation.py (repetition_penalty,
no_repeat_ngram_size, min_length / min_new_tokens, num_return_sequences) against transformers' own processors and
`generate`, and of the reference helper tests/rules_ref.py, which must catch seeded defects."""
import pytest
import torch

from rules_ref import mismatches
from slamkit_b200 import generation as G


def test_rules_equal_hf_processors():
    for V, seed in ((64, 0), (64, 1), (257, 2)):
        assert mismatches(G.apply_rules, V, seed) == []


def test_min_step():
    assert G.min_step(6, None, 3) == 3 and G.min_step(6, 20, 2) == 2 and G.min_step(6, 8, None) == 2
    assert G.min_step(6, 4, None) == 0 and G.min_step(6, None, None) == 0


# seeded defects the helper has to catch
def _penalty_twice(s, **kw):
    s = G.apply_rules(s, **kw)
    p = kw.get("repetition_penalty")
    if p is not None and p != 1.0:
        ids = torch.tensor(sorted(set(kw["history"])), dtype=torch.long)
        g = s[ids]
        s[ids] = torch.where(g < 0, g * p, g / p)
    return s


def _bound_lt_instead_of_le(s, **kw):
    # masks eos while step <= bound instead of step < bound
    s = G.apply_rules(s, **kw)
    step, bound = len(kw["history"]) - kw["prompt_len"], G.min_step(kw["prompt_len"], kw["min_length"], kw["min_new_tokens"])
    if kw["eos"] and step == bound:
        s[list(kw["eos"])] = float("-inf")
    return s


def _ngram_without_pads(s, **kw):
    n = kw.get("no_repeat_ngram_size") or 0
    if n <= 0:
        return G.apply_rules(s, **kw)
    hist = [t for t in kw["history"] if t != 0]
    s = G.apply_rules(s, **dict(kw, no_repeat_ngram_size=0))
    b = G.ngram_bans(hist, n)
    if b:
        s[b] = float("-inf")
    return s


@pytest.mark.parametrize("defect", [_penalty_twice, _bound_lt_instead_of_le, _ngram_without_pads])
def test_helper_catches_defects(defect):
    assert mismatches(defect), defect.__name__


# ------------------------------------------------------------------------------------------ generate_tokens vs HF
@pytest.fixture(scope="module")
def tiny_hf():
    from transformers import Qwen2Config, Qwen2ForCausalLM
    torch.manual_seed(3)
    cfg = Qwen2Config(vocab_size=64, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=1, max_position_embeddings=256, tie_word_embeddings=True, pad_token_id=0,
                      bos_token_id=1, eos_token_id=1)
    return Qwen2ForCausalLM(cfg).eval()


def _batch(V=64):
    g = torch.Generator().manual_seed(5)
    ids, mask = torch.zeros(2, 9, dtype=torch.long), torch.zeros(2, 9, dtype=torch.long)
    ids[0], mask[0] = torch.randint(2, V, (9,), generator=g), 1
    ids[1, 4:], mask[1, 4:] = torch.randint(2, V, (5,), generator=g), 1
    return ids, mask


def _next_logits(m):
    def f(x):
        with torch.no_grad():
            return m(input_ids=x).logits[0, -1]
    return f


RULES = {
    "penalty": dict(repetition_penalty=1.8),
    "penalty<1": dict(repetition_penalty=0.6),
    "ngram1": dict(no_repeat_ngram_size=1),
    "ngram2": dict(no_repeat_ngram_size=2),
    "ngram3-penalty": dict(no_repeat_ngram_size=3, repetition_penalty=1.3),
    "min_new_tokens": dict(min_new_tokens=6, eos="first"),
    "min_length": dict(min_length=14, eos="first"),
}


@pytest.mark.parametrize("case", list(RULES))
def test_greedy_generate_tokens_equals_hf(tiny_hf, case):
    ids, mask = _batch()
    kw = dict(RULES[case])
    eos = None
    if kw.pop("eos", None):
        with torch.no_grad():
            plain = tiny_hf.generate(input_ids=ids, attention_mask=mask, do_sample=False, max_new_tokens=12,
                                     eos_token_id=None, pad_token_id=0)
        eos = int(plain[0, 9])                  # row 0's first greedy token: masked until the bound
    with torch.no_grad():
        want = tiny_hf.generate(input_ids=ids, attention_mask=mask, do_sample=False, max_new_tokens=12, eos_token_id=eos,
                                pad_token_id=0, **kw)
    got = G.generate_tokens(_next_logits(tiny_hf), ids, attention_mask=mask, do_sample=False, max_new_tokens=12,
                            eos_token_id=eos, pad_token_id=0, **kw)
    assert torch.equal(got, want), (case, got, want)


@pytest.mark.parametrize("k", [1, 3])
def test_seeded_sampling_equals_hf(tiny_hf, k):
    ids, mask = _batch()
    kw = dict(do_sample=True, temperature=0.9, top_k=20, max_new_tokens=10, eos_token_id=None, pad_token_id=0,
              repetition_penalty=1.4, no_repeat_ngram_size=2, num_return_sequences=k)
    torch.manual_seed(11)
    with torch.no_grad():
        want = tiny_hf.generate(input_ids=ids, attention_mask=mask, **kw)
    got = G.generate_tokens(_next_logits(tiny_hf), ids, attention_mask=mask, generator=torch.Generator().manual_seed(11),
                            **kw)
    assert got.shape == (2 * k, 19) and torch.equal(got, want), (got, want)
    assert torch.equal(got[:, :9], ids.repeat_interleave(k, 0))


def test_defaults_keep_results_and_greedy_k_raises(tiny_hf):
    ids, mask = _batch()
    f = _next_logits(tiny_hf)
    base = G.generate_tokens(f, ids, attention_mask=mask, max_new_tokens=6, pad_token_id=0)
    same = G.generate_tokens(f, ids, attention_mask=mask, max_new_tokens=6, pad_token_id=0, repetition_penalty=1.0,
                             no_repeat_ngram_size=0, num_return_sequences=1, min_length=0, min_new_tokens=None)
    assert torch.equal(base, same)
    with pytest.raises(ValueError, match="num_return_sequences"):
        G.generate_tokens(f, ids, attention_mask=mask, max_new_tokens=2, num_return_sequences=2)
    with pytest.raises(ValueError, match="strictly positive"):
        G.generate_tokens(f, ids, attention_mask=mask, max_new_tokens=2, repetition_penalty=0.0)
