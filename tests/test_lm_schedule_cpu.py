"""The launch schedule of lm_step.cu, the host side of every decoder the GPU path runs, recorded without a GPU.

lm_step.cu is compiled for sm_90a as it is built into the library, then linked against stubs instead of the kernels and
the CUDA runtime: every launcher of kernels.h it calls prints its name and arguments (pointers as <buffer>+<offset> of a
named buffer), and the runtime stub serves cudaMalloc / cudaMemcpy from host memory and logs the memsets and event
records.  tests/lm_schedule/driver.cpp runs Qwen2, GPT-NeoX and OPT (pre-LN, fp32 master weights, fp32 inference,
post-LN with and without project_in / project_out) through creation, forward, forward-backward, the DPO rows pair,
generation, the optimiser step and the calls each handle refuses.

The same launches with the same arguments and workspace offsets mean the same results and the same speed, so any
change to lm_step.cu that is meant to keep both must leave tests/golden/lm_schedule.txt as it is.  The golden keeps, per
variant and phase (create, forward, training, ...), the number of lines the phase printed and their SHA-256: the calls,
their return codes and refusal messages, every launch with its arguments.  `--full` prints the whole trace.
"""
import hashlib
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "slamkit_b200", "csrc")
HERE = os.path.join(ROOT, "tests", "lm_schedule")
GOLDEN = os.path.join(ROOT, "tests", "golden", "lm_schedule.txt")
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)

# answered by runtime.cpp with fixed values
SIZE_QUERIES = {"sk_gemm_ws_min_bytes", "sk_ce_blocks", "sk_colsum_splits", "sk_rmsnorm_bwd_blocks",
                "sk_layernorm_bwd_blocks"}
INTEGERS = {"int", "long", "size_t", "int32_t", "int64_t", "uint32_t", "unsigned", "bool"}


def _strip_comments(src):
    return re.sub(r"//[^\n]*", "", src)


def _params(plist):
    """[(type, name)] of a declaration's parameter list, defaults dropped."""
    out = []
    for p in plist.split(","):
        p = p.split("=")[0].strip()
        if not p or p == "void":
            continue
        m = re.match(r"(.*?)([A-Za-z_]\w*)$", p)
        out.append((m.group(1).strip(), m.group(2)))
    return out


def _fmt(ty, name):
    """printf conversion and argument for one parameter"""
    if "*" in ty or ty == "cudaStream_t":
        return "%s", f"tr_ptr((const void*){name})"
    if ty in ("float", "double"):
        return "%.9g", f"(double){name}"
    base = ty.replace("const", "").strip()
    assert base in INTEGERS, f"launcher parameter of unknown type: {ty} {name}"
    return "%lld", f"(long long){name}"


def _gemm_ex_fields(header):
    body = re.search(r"struct SkGemmEx \{(.*?)\n\};", header, re.S).group(1)
    fields = []
    for stmt in body.split(";"):
        stmt = stmt.strip()
        if not stmt:
            continue
        m = re.match(r"((?:const\s+)?\w+\**)\s*(.*)$", stmt, re.S)
        ty, names = m.group(1), m.group(2)
        for nm in names.split(","):
            nm = nm.strip()
            fields.append(("void*" if nm.startswith("*") else ty, nm.lstrip("*")))
    return fields


def launcher_stubs():
    """kernels.h's launchers that lm_step.cu calls, each defined to print its arguments"""
    header = _strip_comments(open(os.path.join(CSRC, "kernels.h")).read())
    used = set(re.findall(r"\b(sk_\w+)\s*\(", open(os.path.join(CSRC, "lm_step.cu")).read()))
    used.add("sk_gemm_ex_launch")   # the launcher behind every GEMM descriptor builder
    out = ['#include "kernels.h"', '#include "trace.h"', ""]
    decls = re.finditer(r"^(extern \"C\" )?(int|size_t|SkGemmEx)\s+(sk_\w+)\(([^)]*)\)\s*;", header, re.M)
    for m in decls:
        ret, name, plist = m.group(2), m.group(3), m.group(4)
        if m.group(1) or name not in used or name in SIZE_QUERIES:
            continue
        params = _params(plist)
        sig = ", ".join(f"{t} {n}" for t, n in params)
        lines = [f"{ret} {name}({sig}) {{"]
        if name == "sk_gemm_ex_launch":
            g = params[0][1]
            fs = [(_fmt(t, f"{g}.{f}"), f) for t, f in _gemm_ex_fields(header)]
            fmt = " ".join(f"{f}=%s" if c == "%s" else f"{f}={c}" for (c, _), f in fs)
            args = ", ".join(a for (_, a), _ in fs)
            lines.append(f'  tr_log("{name}({fmt}, %s)", {args}, tr_ptr({params[1][1]}));')
        else:
            convs = [_fmt(t, n) for t, n in params]
            fmt = ", ".join(c for c, _ in convs)
            args = ", ".join(a for _, a in convs)
            lines.append(f'  tr_log("{name}({fmt})", {args});')
        names = {n for _, n in params}
        if {"chunk_start", "chunk_len", "n_chunks"} <= names:
            # the chunk tables live in host memory here (runtime.cpp's cudaMalloc)
            lines.append('  for (int i = 0; i < n_chunks; ++i) tr_log("  chunk %ld %d", chunk_start[i], chunk_len[i]);')
        if {"tensor_chunk_begin", "n_tensors"} <= names:
            lines.append('  for (int i = 0; i <= n_tensors; ++i) tr_log("  group %d", tensor_chunk_begin[i]);')
        lines += ["  return 0;", "}", ""]
        out += lines
    return "\n".join(out)


def build_tracer(tmp):
    gen = os.path.join(tmp, "launchers.cu")
    with open(gen, "w") as f:
        f.write(launcher_stubs())
    nv = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-Xcompiler", "-fPIC",
          "--expt-relaxed-constexpr", "-I", CSRC, "-I", HERE, "-c"]
    cxx = ["g++", "-O1", "-std=c++17", "-I", HERE, "-c"]
    jobs = [nv + [os.path.join(CSRC, "lm_step.cu"), "-o", os.path.join(tmp, "lm_step.o")],
            nv + [gen, "-o", os.path.join(tmp, "launchers.o")],
            cxx + [os.path.join(HERE, "runtime.cpp"), "-o", os.path.join(tmp, "runtime.o")],
            cxx + [os.path.join(HERE, "driver.cpp"), "-o", os.path.join(tmp, "driver.o")]]
    procs = [subprocess.Popen(j, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for j in jobs]
    for j, p in zip(jobs, procs):
        out = p.communicate()[0]
        assert p.returncode == 0, f"{' '.join(j)}\n{out}"
    exe = os.path.join(tmp, "lm_schedule")
    subprocess.run(["g++", "-o", exe] + [os.path.join(tmp, o) for o in
                                         ("driver.o", "lm_step.o", "launchers.o", "runtime.o")], check=True)
    return exe


def trace(tmp):
    env = {k: v for k, v in os.environ.items() if k != "SK_HEAD_CHUNK"}
    return subprocess.run([build_tracer(tmp)], check=True, capture_output=True, text=True, env=env).stdout


def phases(text):
    """[(name, lines)]: the trace cut at the driver's phase markers, "<variant>: create" (creation and binding), then
    "<variant>: forward", "training" and so on, each with every line it printed (calls, return codes, launches)."""
    out = []
    for ln in text.splitlines():
        if ln.startswith("==== "):
            variant = ln[5:]
            out.append([variant + ": create", []])
        elif ln.startswith("## "):
            out.append([f"{variant}: {ln[3:]}", []])
        else:
            out[-1][1].append(ln)
    return out


def digest(text):
    """The golden form of a trace: per phase its name, the number of lines it printed and their SHA-256 (16 hex)."""
    return "".join(f"{name} | {len(b)} {hashlib.sha256(chr(10).join(b).encode()).hexdigest()[:16]}\n"
                   for name, b in phases(text))


@pytest.mark.skipif(NVCC is None or shutil.which("g++") is None, reason="needs nvcc and g++")
def test_launch_schedule_matches_golden(tmp_path):
    got = trace(str(tmp_path))
    unresolved = [ln for ln in got.splitlines() if re.search(r"(^|[ (=,])\?([,) ]|$)", ln)]
    assert not unresolved, "pointers outside every named buffer:\n" + "\n".join(unresolved[:20])
    g, w = digest(got).splitlines(), open(GOLDEN).read().splitlines()
    if g != w:
        i = next((k for k in range(min(len(g), len(w))) if g[k] != w[k]), min(len(g), len(w)))
        now = "\n".join("    " + ln for ln in phases(got)[i][1]) if i < len(g) else ""
        pytest.fail(f"launch schedule differs from {os.path.relpath(GOLDEN, ROOT)}:\n"
                    f"  golden: {w[i] if i < len(w) else '<end>'}\n  now:    {g[i] if i < len(g) else '<end>'}\n"
                    f"  what this phase prints now (compare with `python {os.path.relpath(__file__, ROOT)} --full` "
                    f"on the parent commit):\n{now}")


if __name__ == "__main__":
    # python tests/test_lm_schedule_cpu.py          the golden digest (tests/golden/lm_schedule.txt)
    # python tests/test_lm_schedule_cpu.py --full   the whole trace, to compare two builds line by line
    import sys
    import tempfile

    with tempfile.TemporaryDirectory() as d:
        t = trace(d)
        sys.stdout.write(t if "--full" in sys.argv else digest(t))
