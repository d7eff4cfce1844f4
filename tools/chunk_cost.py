"""Cost of the memory-bounded (chunked) layer search on the GPU.

  python tools/chunk_cost.py [--repeats 3] [--out FILE.json]

1. ViT-B/224 x 32 images, qkv (normal-equation weight steps), fc2 (post-GELU) and matmul2 (split-of-softmax), searched
   whole and in 2 and 4 chunks: one
   warm-up search per setting, then the settings alternated `--repeats` times; each search is timed by the host clock
   around a device synchronise.  The step sizes of every setting are compared with the whole-layer search.
2. DeiT-B/384 x 128 images, fc2 and matmul2 under a 20 GiB workspace budget (their whole-layer workspaces are 23 GB and
   61 GB), qkv whole (17 GB) and under an 8 GiB budget: wall time, peak device memory besides the captured tensors, and
   whether the step sizes equal those of the whole-layer search (qkv).

W8A8, n_V = n_H = 24 (qkv: n_V = 72), eq_n = 100, three search rounds, hessian metric, as bench.py's default workload.
Chunking is forced through P4V_WORKSPACE_BUDGET.  Prints one JSON document (also written to --out)."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ptq4vit_b200 import _lib  # noqa: E402
from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLBatchingQuantLinear, PTQSLBatchingQuantLinear  # noqa: E402
from ptq4vit_b200.quant_layers.matmul import SoSPTQSLBatchingQuantMatMul  # noqa: E402

KW = dict(metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=3)


def gpu_state():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def fc2(n_img, tok, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.nn.functional.gelu(torch.randn(n_img, tok, 3072, device="cuda", generator=gen) * 1.5)
    m = PostGeluPTQSLBatchingQuantLinear(3072, 768, n_V=24, n_H=24, n_a=1, **KW).cuda()
    with torch.no_grad():
        y = m(x)
    g = torch.randn(y.shape, device="cuda", generator=gen) * 1e-3
    return m, (x, y, g)


def qkv(n_img, tok, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n_img, tok, 768, device="cuda", generator=gen)
    m = PTQSLBatchingQuantLinear(768, 2304, n_V=72, n_H=24, n_a=1, **KW).cuda()
    with torch.no_grad():
        y = m(x)
    g = torch.randn(y.shape, device="cuda", generator=gen) * 1e-3
    return m, (x, y, g)


def matmul2(n_img, tok, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.softmax(torch.randn(n_img, 12, tok, tok, device="cuda", generator=gen) * 4.0, dim=-1)
    B = torch.randn(n_img, 12, tok, 64, device="cuda", generator=gen)
    Y = A @ B
    G = torch.randn(Y.shape, device="cuda", generator=gen) * 1e-3
    return SoSPTQSLBatchingQuantMatMul(**KW), (A, B, Y, G)


def search(m, t):
    if isinstance(m, SoSPTQSLBatchingQuantMatMul):
        m.raw_input, m.raw_out, m.raw_grad = [t[0], t[1]], t[2], t[3]
    else:
        m.raw_input, m.raw_out, m.raw_grad = t
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    vals = (m.A_interval, m.B_interval, m.split) if isinstance(m, SoSPTQSLBatchingQuantMatMul) else (m.w_interval, m.a_interval)
    return dt, [torch.as_tensor(v).detach().float().cpu().reshape(-1) for v in vals]


def budget_for(m, t, k):
    """Workspace bytes of the module's search in k chunks (k = 1: the whole layer)."""
    n = ctypes.c_size_t()
    if isinstance(m, SoSPTQSLBatchingQuantMatMul):
        d = m._desc(t[0], t[1], m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
        d.images_per_chunk = 0 if k == 1 else -(-d.batch // k)
        _lib.check(_lib.lib().p4v_matmul_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "workspace")
    else:
        rows, tok = t[0].shape[0] * t[0].shape[1], t[0].shape[1]
        d = m._desc(rows, tok, m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
        d.rows_per_chunk = 0 if k == 1 else -(-(-(-rows // k)) // 128) * 128
        _lib.check(_lib.lib().p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "workspace")
    return n.value


def chunk_cost(name, make, repeats):
    m, t = make(32, 197, 1)
    ks = (1, 2, 4)
    budgets = {k: budget_for(m, t, k) for k in ks}
    times = {k: [] for k in ks}
    ref = None
    same = True
    for rep in range(repeats + 1):          # round 0 warms every setting up
        for k in ks:
            os.environ["P4V_WORKSPACE_BUDGET"] = str(budgets[k])
            dt, vals = search(m, t)
            assert m.calib_chunks == k
            if ref is None:
                ref = vals
            same = same and all(torch.equal(a, b) for a, b in zip(ref, vals))
            if rep > 0:
                times[k].append(dt)
    os.environ.pop("P4V_WORKSPACE_BUDGET", None)
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"layer": name, "workspace_bytes": budgets, "search_s": times, "median_s": med,
            "slowdown_vs_whole": {k: med[k] / med[1] for k in ks}, "step_sizes_identical": bool(same)}


def budgeted(name, make, budgets):
    """One search per budget (None: the free device memory) after a warm-up, twice, alternated."""
    m, t = make(128, 577, 2)
    captures = sum(v.numel() * v.element_size() for v in t)
    out = {b: {"search_s": []} for b in budgets}
    for rep in range(3):                     # round 0 warms up
        for b in budgets:
            if b is None:
                os.environ.pop("P4V_WORKSPACE_BUDGET", None)
            else:
                os.environ["P4V_WORKSPACE_BUDGET"] = str(b)
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            dt, vals = search(m, t)
            r = out[b]
            r.update(chunks=m.calib_chunks, peak_bytes_besides_captures=torch.cuda.max_memory_allocated() - base,
                     step_sizes=vals)
            if rep > 0:
                r["search_s"].append(dt)
    os.environ.pop("P4V_WORKSPACE_BUDGET", None)
    ref = out[budgets[0]]["step_sizes"]
    res = []
    for b in budgets:
        r = out[b]
        same = all(torch.equal(x, y) for x, y in zip(ref, r.pop("step_sizes")))
        res.append({"layer": name, "budget_bytes": b, "captured_bytes": captures, "step_sizes_equal_first": bool(same), **r})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/chunk_cost.py measures on the GPU"
    res = {"gpu_before": gpu_state(), "config": "W8A8, fc2 n_V=n_H=24, eq_n=100, 3 rounds, hessian"}
    res["vitb224x32"] = [chunk_cost("qkv", qkv, a.repeats), chunk_cost("fc2", fc2, a.repeats),
                         chunk_cost("matmul2", matmul2, a.repeats)]
    torch.cuda.empty_cache()
    res["deitb384x128"] = []
    for name, make, budgets in (("matmul2", matmul2, [20 << 30]), ("fc2", fc2, [20 << 30]), ("qkv", qkv, [None, 8 << 30])):
        res["deitb384x128"] += budgeted(name, make, budgets)
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_state()
    text = json.dumps(res, indent=1, default=str)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
