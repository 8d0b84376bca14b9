"""The GEMM planner's choices on the H100's 132 SMs, asked through the C ABI (sk_gemm_plan: nothing is launched and no
pointer is dereferenced, so this runs without a GPU, where the SM count falls back to 132).

- The 12 GEMMs of a cfg-2 layer (Qwen2.5-0.5B shape, 8 x 1024 tokens) take the tile widths that fit the model:
  224 for d = 896 and 192 for QKV = 1152 where no stream-K scratch is given (forward and dgrad), and column-unit
  stream-K for the down-projection weight gradient.
- The decode and OPT shapes plan exactly as they did before the 192 / 224 widths existed
  (tests/golden/gemm_plans_h100.json, recorded on an H100 SXM).
"""
import ctypes as C
import json
import os

import pytest

from slamkit_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
FIELDS = [f for f, _ in L.SkGemmPlan._fields_]


@pytest.fixture(scope="module")
def lib():
    lib = L.load()
    if lib.sk_device_sm_count() != 132:
        pytest.skip("the plan tables are for 132 SMs (H100 SXM)")
    return lib


def _plan(lib, M, N, K, a_mn=0, b_mn=0, bias=0, res=None, rbr=0, act=0, ws=0, force_bn=0):
    fake = lambda i: C.c_void_p((i + 1) << 32)   # distinct, 16-byte aligned, never dereferenced
    c = fake(2)
    r = c if res == "inplace" else (fake(4) if res else C.c_void_p(0))
    ws_bytes = int(lib.sk_gemm_ws_bytes()) + (64 << 20) if ws else 0
    p = L.SkGemmPlan()
    rc = lib.sk_gemm_plan(M, N, K, fake(0), M if a_mn else K, a_mn, fake(1), N if b_mn else K, b_mn, c, N, 0,
                          fake(3) if bias else C.c_void_p(0), r, N if res else 0, rbr, act, force_bn,
                          fake(9) if ws else C.c_void_p(0), C.c_int64(ws_bytes), C.byref(p))
    assert rc == 0, lib.sk_last_error().decode()
    return {f: int(getattr(p, f)) for f in FIELDS}


T, d, F, Q = 8192, 896, 4864, 1152
# name -> (plan arguments, expected: bn, schedule)   schedule: plain / splitk / rows / cols (row- / column-unit stream-K)
CFG2 = {
    "qkv_fwd": (dict(M=T, N=Q, K=d, bias=1), 192, "plain"),
    "o_fwd": (dict(M=T, N=d, K=d, res=1, rbr=1), 224, "plain"),
    "gu_fwd": (dict(M=T, N=2 * F, K=d), 256, "plain"),
    "down_fwd": (dict(M=T, N=d, K=F, res=1, rbr=1), 224, "plain"),
    "down_dgrad": (dict(M=T, N=F, K=d, b_mn=1), 256, "plain"),
    "gu_dgrad": (dict(M=T, N=d, K=2 * F, b_mn=1), 224, "plain"),
    "o_dgrad": (dict(M=T, N=d, K=d, b_mn=1), 224, "plain"),
    "qkv_dgrad": (dict(M=T, N=d, K=Q, b_mn=1), 224, "plain"),
    "down_wgrad": (dict(M=d, N=F, K=T, a_mn=1, b_mn=1, ws=1), 256, "cols"),
    "gu_wgrad": (dict(M=2 * F, N=d, K=T, a_mn=1, b_mn=1, ws=1), 256, "rows"),
    "o_wgrad": (dict(M=d, N=d, K=T, a_mn=1, b_mn=1, ws=1), 128, "splitk"),
    "qkv_wgrad": (dict(M=Q, N=d, K=T, a_mn=1, b_mn=1, ws=1), 128, "splitk"),
}


def _schedule(p):
    if p["splits"] > 1:
        return "splitk"
    if p["sk_units"] > 0:
        return "cols" if p["sk_colunits"] else "rows"
    return "plain"


@pytest.mark.parametrize("name", list(CFG2))
def test_cfg2_layer_plans(lib, name):
    args, bn, sched = CFG2[name]
    p = _plan(lib, **args)
    assert (p["bn"], _schedule(p)) == (bn, sched), p


def test_down_wgrad_streamk_balance(lib):
    """7 x 19 tiles of 256: 19 column units over 18 groups of 7 CTAs; the last full wave and the leftover unit are laid
    end to end, so every group runs 19/18 of a unit and each unit is cut into at most two ranges."""
    p = _plan(lib, **CFG2["down_wgrad"][0])
    assert (p["sk_units"], p["sk_groups"], p["sk_G"], p["grid"]) == (19, 18, 7, 126), p
    num_kb = T // 64
    starts = [p["sk_units"] * num_kb * g // p["sk_groups"] for g in range(p["sk_groups"])]
    inside = [sum(1 for s in starts if u * num_kb < s < (u + 1) * num_kb) for u in range(p["sk_units"])]
    assert max(inside) == 1, inside


def test_forced_widths(lib):
    """force_bn takes 192 and 224 as it takes 64 / 128 / 256, on any N."""
    for bn in (64, 128, 192, 224, 256):
        assert _plan(lib, M=1000, N=1000, K=512, force_bn=bn)["bn"] == bn


def test_decode_and_opt_plans_unchanged(lib):
    golden = json.load(open(os.path.join(HERE, "golden", "gemm_plans_h100.json")))
    changed = {k: (v["plan"], _plan(lib, **v["args"])) for k, v in golden.items() if _plan(lib, **v["args"]) != v["plan"]}
    assert not changed, changed
