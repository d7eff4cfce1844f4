"""Time the quantised forward of a calibrated ViT-B/224 on one GPU, unfrozen against frozen, and print one JSON line.

    python tools/forward_bench.py [--images 32] [--bit 8] [--reps 3] [--window 1.0]

Workload: synthetic weights, a seeded calibration on `--images` synthetic 224x224 images (HessianQuantCalibrator), then
an evaluation batch of 32 images, W{bit}A{bit}, for the PTQ4ViT configuration (n_H = 24) and BasePTQ (n_H = 1, Hessian
metric).  After a warm-up of every shape, `--reps` times alternately:

  (a) today's quant_forward (weight and activation images rebuilt per call), (b) the frozen forward

per module type (qkv, proj, fc1, fc2, head, matmul1, matmul2; one module of each, its real input from the quantised
model -- for the MatMul modules the strided q / k^T / v views themselves) with CUDA events over enough calls to fill
`--window` seconds; then the 49 Linear modules of the model in sequence on their own inputs -- (a), (b) and (b) replayed
from one CUDA graph -- and the whole quantised model forward, host clock around a device synchronise: unfrozen, Linear
frozen (`freeze_model(wrapped)`), Linear and MatMul frozen (`freeze_model(wrapped, matmul=True)`), and the latter
replayed from one CUDA graph of the whole forward.  The per-type (b) of the MatMul modules is their frozen forward.

Per module type the output also has the bytes a call must move (Linear: FP32 x, int8 weight, FP32 out; MatMul: FP32 A,
B and out) and its integer operations (2 * rows * in * out per activation part; MatMul 2 * S1 * S2 * S3 per problem and
A part), both from the shapes, the HBM bound of those bytes at the H100 SXM data sheet's 3.35 TB/s and the share of it
the frozen forward reaches.  The card, its power limit and its max SM clock
come from one read-only nvidia-smi query.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import importlib
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TQDM_DISABLE", "1")

import torch  # noqa: E402

MODEL = "vit_base_patch16_224"
TYPES = ("qkv", "proj", "fc1", "fc2", "head")
MM_TYPES = ("matmul1", "matmul2")
HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, power, sm = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit_w": float(power), "max_sm_mhz": float(sm)}


def calibrated_model(config, images, bit):
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import get_net
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    cfg = importlib.import_module(f"ptq4vit_b200.configs.{config}")
    importlib.reload(cfg)
    if config == "BasePTQ":
        for d in (cfg.ptqsl_conv2d_kwargs, cfg.ptqsl_linear_kwargs, cfg.ptqsl_matmul_kwargs):
            d["metric"] = "hessian"
    for d in (cfg.w_bit, cfg.a_bit, cfg.A_bit, cfg.B_bit):
        for k in d:
            d[k] = bit
    net = get_net(MODEL, device=torch.device("cuda", 0), seed=0)
    wrapped = wrap_modules_in_net(net, cfg)
    calib = torch.randn(images, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    Q.HessianQuantCalibrator(net, wrapped, [(calib, None)], sequential=False, batch_size=4, target_noise=1.0).batching_quant_calib()
    torch.cuda.synchronize()
    return net, wrapped


def capture_inputs(net, linear, batch, matmuls=()):
    """The input of every Linear module (and of the given MatMul modules: both operands, as the strided views they are
    called with) in one quantised forward of the evaluation batch."""
    inputs, hooks = {}, []
    for name, m in linear.items():
        hooks.append(m.register_forward_pre_hook(lambda mod, inp, name=name: inputs.__setitem__(name, inp[0].detach().contiguous())))
    for name, m in matmuls:
        hooks.append(m.register_forward_pre_hook(lambda mod, inp, name=name: inputs.__setitem__(name, (inp[0].detach(), inp[1].detach()))))
    with torch.no_grad():
        net(batch)
    for h in hooks:
        h.remove()
    torch.cuda.synchronize()
    return inputs


def events_ms(fn, window_s):
    """Mean ms per call over enough calls to fill window_s (CUDA events)."""
    def run(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    n = max(10, int(math.ceil(window_s * 1e3 / max(run(10), 1e-3))))
    return run(n), n


def wall_ms(fn, window_s):
    """Mean wall ms per call, host clock around a device synchronise."""
    def run(n):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n
    n = max(3, int(math.ceil(window_s * 1e3 / max(run(2), 1e-3))))
    return run(n), n


def bench_config(config, a):
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul
    from ptq4vit_b200.utils import deploy
    net, wrapped = calibrated_model(config, a.images, a.bit)
    linear = {n: m for n, m in wrapped.items() if isinstance(m, MinMaxQuantLinear)}
    mm_one = {t: next(n for n, m in wrapped.items() if isinstance(m, MinMaxQuantMatMul) and n.endswith(t)) for t in MM_TYPES}
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    inputs = capture_inputs(net, linear, batch, [(mm_one[t], wrapped[mm_one[t]]) for t in MM_TYPES])
    one = {t: next(n for n in linear if n.rsplit(".", 1)[-1] == t) for t in TYPES}
    one.update(mm_one)
    mods = {t: wrapped[one[t]] for t in TYPES + MM_TYPES}

    def call(t):
        x = inputs[one[t]]
        return mods[t].quant_forward(*x) if t in MM_TYPES else mods[t].quant_forward(x)

    def set_frozen(mode):
        """None: nothing frozen; "linear": the Linear modules; "all": Linear and MatMul modules."""
        deploy.unfreeze_model(wrapped)
        if mode:
            deploy.freeze_model(wrapped, matmul=mode == "all")

    def chain():
        for n, m in linear.items():
            m.quant_forward(inputs[n])

    def model():
        net(batch)

    alive = []

    def graph_of(fn):
        """fn captured in a CUDA graph.  The graph reads the packed tensors (and the streamed Linear workspace) of the
        current freeze: they are kept alive here, since set_frozen() drops the modules' references."""
        fn()
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()
        torch.cuda.current_stream().wait_stream(side)
        with torch.cuda.graph(graph):
            fn()
        graph.replay()
        alive.extend((getattr(m, "_packed", None), getattr(m, "_frozen_ws", None)) for m in wrapped.values())
        return graph

    bits = lambda t: t.contiguous().view(torch.int32)
    # outputs must not change, at the sizes timed
    with torch.no_grad():
        want = {t: call(t) for t in TYPES + MM_TYPES}
        logits = net(batch)
        set_frozen("linear")
        identical = all(torch.equal(bits(call(t)), bits(want[t])) for t in TYPES) and torch.equal(bits(net(batch)), bits(logits))
        paths = {t: "fused" if mods[t]._frozen_fused else "streamed" for t in TYPES}
        graph = graph_of(chain)                   # warm-up of every shape, Linear frozen ...
        set_frozen("all")
        identical_all = all(torch.equal(bits(call(t)), bits(want[t])) for t in TYPES + MM_TYPES) and \
            torch.equal(bits(net(batch)), bits(logits))
        model_graph = graph_of(model)             # ... everything frozen: the whole forward in one graph ...
        model_graph.replay(); torch.cuda.synchronize()
        logits_graph = net(batch)
        identical_graph = torch.equal(bits(logits_graph), bits(logits))
        set_frozen(None)
        chain(); model()                          # ... and unfrozen
        torch.cuda.synchronize()

        per = {t: {"unfrozen_ms": [], "frozen_ms": []} for t in TYPES + MM_TYPES}
        whole = {"linear_chain_unfrozen_ms": [], "linear_chain_frozen_ms": [], "linear_chain_frozen_graph_ms": [],
                 "model_unfrozen_ms": [], "model_frozen_ms": [], "model_frozen_with_matmul_ms": [],
                 "model_frozen_with_matmul_graph_ms": []}
        calls = {}
        for _ in range(a.reps):
            for mode in (None, "linear", "all"):
                set_frozen(mode)
                key = "frozen_ms" if mode else "unfrozen_ms"
                for t in (TYPES + MM_TYPES if mode is None else TYPES if mode == "linear" else MM_TYPES):
                    ms, calls[f"{t}_{key}"] = events_ms(lambda: call(t), a.window)
                    per[t][key].append(ms)
                if mode == "all":
                    whole["model_frozen_with_matmul_ms"].append(wall_ms(model, a.window)[0])
                    continue
                tag = "frozen" if mode else "unfrozen"
                whole[f"linear_chain_{tag}_ms"].append(wall_ms(chain, a.window)[0])
                whole[f"model_{tag}_ms"].append(wall_ms(model, a.window)[0])
            whole["linear_chain_frozen_graph_ms"].append(wall_ms(graph.replay, a.window)[0])
            whole["model_frozen_with_matmul_graph_ms"].append(wall_ms(model_graph.replay, a.window)[0])
        set_frozen(None)

    out = {"config": config, "bit_identical": bool(identical), "bit_identical_with_matmul": bool(identical_all),
           "bit_identical_model_graph": bool(identical_graph), "linear_modules": len(linear), "per_type": {},
           "calls_per_window": calls}
    for t in TYPES + MM_TYPES:
        m = mods[t]
        if t in MM_TYPES:
            A, B = inputs[one[t]]
            (b, H, S1, S2), S3 = A.shape, B.shape[3]
            nbytes = 4 * b * H * (S1 * S2 + S2 * S3 + S1 * S3)
            entry = {"A": list(A.shape), "B": list(B.shape), "A_strides": list(A.stride()), "B_strides": list(B.stride()),
                     "class": type(m).__name__, "int_ops": 2 * b * H * S1 * S2 * S3 * (2 if m.sos else 1)}
        else:
            x = inputs[one[t]]
            rows, K, O = x.numel() // x.shape[-1], m.in_features, m.out_features
            parts = 2 if m.post_gelu else 1
            nbytes = rows * K * 4 + O * K + rows * O * 4
            entry = {"rows": rows, "in": K, "out": O, "path": paths[t], "int_ops": 2 * rows * K * O * parts}
        u, f = statistics.median(per[t]["unfrozen_ms"]), statistics.median(per[t]["frozen_ms"])
        bound_ms = nbytes / HBM_BYTES_PER_S * 1e3
        out["per_type"][t] = {**entry, "bytes": nbytes, "hbm_bound_ms": round(bound_ms, 4),
                              "unfrozen_ms": round(u, 4), "frozen_ms": round(f, 4), "speedup": round(u / f, 2),
                              "frozen_share_of_hbm_bound": round(bound_ms / f, 3),
                              "unfrozen_runs_ms": [round(v, 4) for v in per[t]["unfrozen_ms"]],
                              "frozen_runs_ms": [round(v, 4) for v in per[t]["frozen_ms"]]}
    out["whole"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}
    del net, wrapped, linear, inputs, graph, model_graph, mods, alive
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32, help="calibration images")
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timing")
    ap.add_argument("--configs", default="PTQ4ViT,BasePTQ")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/forward_bench.py needs a CUDA device (no CPU fallback)")
    torch.cuda.set_device(0)
    out = {"tool": "forward_bench", "card": card(),
           "workload": f"{MODEL}, synthetic weights, calibrated on {a.images} synthetic imgs, evaluation batch 32, W{a.bit}A{a.bit}",
           "hbm_bytes_per_s_data_sheet": HBM_BYTES_PER_S,
           "configs": [bench_config(c, a) for c in a.configs.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
