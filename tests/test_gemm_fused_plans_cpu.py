"""The GEMM planner's choices for every fused linear and for the plain GEMM, asked through the C ABI without a GPU
(sk_neox_gemm_plan / sk_gemm_plan: nothing is launched and no pointer is dereferenced; the SM count falls back to 132).

Each kind of sk_neox_gemm_plan builds its descriptor with the builder that the launch of that fused linear uses, so the
plans here are the plans of the launches.  tests/golden/gemm_fused_plans.npz holds, for a grid of decode- to
training-sized M and the widths of Qwen2.5-0.5B, Pythia and OPT, every SkGemmPlan field or the refusal message; a
change to a descriptor's pitches, flags or epilogue, or to the planner, shows up as a changed plan.
`PYTHONPATH=. python tests/test_gemm_fused_plans_cpu.py` rewrites the golden from the library in the tree.
"""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

from slamkit_b200 import _lib as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_fused_plans.npz")
FIELDS = [f for f, _ in L.SkGemmPlan._fields_]

MS = (1, 8, 65, 129, 2048, 8192)
# hidden, q|k|v, FFN and gate|up widths of Qwen2.5-0.5B (896, 1152, 4864, 9728), Pythia-70m / -160m / -410m
# (512, 1536, 2048; 768, 2304, 3072; 1024, 3072, 4096) and OPT-125m / -350m (768, 3072; 1024, 4096, project_in 512)
WIDTHS = (512, 768, 896, 1024, 1152, 1536, 2048, 2304, 3072, 4096, 4864, 9728)
KINDS = range(7)
# the plain GEMMs of the LM step, as sk_gemm_plan arguments: (a_mn, b_mn, bias, residual, act)
PLAIN = {"fwd": (0, 0, 0, None, 0), "fwd_bias_res": (0, 0, 1, "other", 0), "fwd_bias_relu": (0, 0, 1, None, 2),
         "dgrad": (0, 1, 0, None, 0), "dgrad_res": (0, 1, 0, "other", 0), "wgrad_acc": (1, 1, 0, "inplace", 0)}


def _fused_plan(lib, kind, M, N, K, ws):
    p = L.SkGemmPlan()
    rc = lib.sk_neox_gemm_plan(kind, M, N, K, ws, C.byref(p))
    return rc, p


def _plain_plan(lib, name, M, N, K, ws):
    a_mn, b_mn, bias, res, act = PLAIN[name]
    fake = lambda i: C.c_void_p((i + 1) << 32)   # distinct, 16-byte aligned, never dereferenced
    c = fake(2)
    r = c if res == "inplace" else (fake(4) if res else C.c_void_p(0))
    p = L.SkGemmPlan()
    rc = lib.sk_gemm_plan(M, N, K, fake(0), M if a_mn else K, a_mn, fake(1), N if b_mn else K, b_mn, c, N, 0,
                          fake(3) if bias else C.c_void_p(0), r, N if res else 0, 1 if res else 0, act, 0,
                          fake(9) if ws else C.c_void_p(0), C.c_int64(int(lib.sk_gemm_ws_bytes()) if ws else 0),
                          C.byref(p))
    return rc, p


def grid():
    for (what, M, N, K, ws) in itertools.product(list(KINDS) + list(PLAIN), MS, WIDTHS, WIDTHS, (0, 1)):
        yield str(what), M, N, K, ws


def record(lib):
    """(case names, plans [n, len(FIELDS)], return codes, refusal messages) over the grid"""
    names, plans, rcs, errs = [], [], [], []
    for what, M, N, K, ws in grid():
        rc, p = (_plain_plan(lib, what, M, N, K, ws) if what in PLAIN else _fused_plan(lib, int(what), M, N, K, ws))
        names.append(f"{what} M={M} N={N} K={K} ws={ws}")
        plans.append([int(getattr(p, f)) if rc == 0 else 0 for f in FIELDS])
        rcs.append(rc)
        errs.append("" if rc == 0 else lib.sk_last_error().decode())
    return np.array(names), np.array(plans, dtype=np.int32), np.array(rcs, dtype=np.int32), np.array(errs)


@pytest.fixture(scope="module")
def lib():
    lib = L.load()
    if lib.sk_device_sm_count() != 132:
        pytest.skip("the plan tables are for 132 SMs (H100 SXM)")
    return lib


def test_plans_match_golden(lib):
    names, plans, rcs, errs = record(lib)
    g = np.load(GOLDEN)
    assert list(g["fields"]) == FIELDS
    assert list(names) == list(g["names"]), "the grid differs from the golden's"
    bad = [f"{n}: golden {list(gp) if grc == 0 else ge!r}, now {list(p) if rc == 0 else e!r}"
           for n, p, rc, e, gp, grc, ge in zip(names, plans, rcs, errs, g["plans"], g["rcs"], g["errs"])
           if (rc != 0) != (grc != 0) or (rc == 0 and list(p) != list(gp)) or (rc != 0 and e != ge)]
    assert not bad, f"{len(bad)} plans differ:\n" + "\n".join(bad[:20])


if __name__ == "__main__":
    names, plans, rcs, errs = record(L.load())
    np.savez_compressed(GOLDEN, fields=np.array(FIELDS), names=names, plans=plans, rcs=rcs, errs=errs)
    print(f"{len(names)} plans, {int((rcs != 0).sum())} refusals -> {GOLDEN}")
