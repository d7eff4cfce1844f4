"""Phase breakdown of the sweep kernel from clocks inside it (GPU box).  usage: sweep_phases.py [layer ...] (default: fc1 qkv)

Builds the library with -DP4V_SWEEP_PHASE_CLOCKS into a temporary directory (the in-tree build is not touched), runs the
search of each ViT-B-shaped layer once to warm up and once measured (the fixtures of tools/profile_layer.py), and prints,
per kernel instantiation that ran, each phase's share of the consumer's (or the producer's) cycles.  Consumer phases are
summed over consumer warp 0 of both warpgroups of every CTA, producer phases over the producer warp; the clock reads
themselves add a little to every phase."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ptq4vit_b200 import build as B  # noqa: E402
from ptq4vit_b200 import _lib  # noqa: E402

KINDS = ["bf16 multi", "bf16 single", "bf16 pair", "int8 multi", "int8 single", "int8 pair"]
CONSUMER = ["wait full", "wgmma wait", "fixed epilogue", "candidate epilogue", "final epilogue + g", "score reduction"]
N_PHASES = 9   # kPh* in csrc/sweep_tc.cu: the six above, consumer total, producer wait on empty, producer total


def build_phase_lib(out_dir):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs, procs = [], []
    for src in B.SOURCES:
        o = os.path.join(out_dir, src.replace(".cu", ".o"))
        objs.append(o)
        cmd = [nvcc] + B.NVCC_FLAGS + ["-DP4V_SWEEP_PHASE_CLOCKS", "-c", os.path.join(B.CSRC, src), "-o", o]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    lib = os.path.join(out_dir, "libptq4vit_b200_phases.so")
    subprocess.check_call([nvcc, "-shared", "-o", lib] + objs + B.GENCODE)
    return lib


def layer_runner(kind, nb=24):
    import torch
    from oracle import ptq_oracle as O  # fixtures only (seeded synthetic tensors)
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear, PostGeluPTQSLBatchingQuantLinear
    D = 768
    K, Oo, nV, gelu = {"qkv": (D, 3 * D, 3 * nb, False), "proj": (D, D, nb, False), "fc1": (D, 4 * D, nb, False),
                       "fc2": (4 * D, D, nb, True)}[kind]
    x, W, b, y, g = O.make_linear_fixture(1, 32, 197, K, Oo, post_gelu=gelu)
    cls = PostGeluPTQSLBatchingQuantLinear if gelu else PTQSLBatchingQuantLinear
    m = cls(K, Oo, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=1, n_V=nV, n_H=nb, n_a=1)
    m.weight.data = W; m.bias.data = b; m.cuda()
    t = [x.cuda(), y.cuda(), g.cuda()]

    def run():
        m.raw_input, m.raw_out, m.raw_grad = t
        with torch.no_grad():
            m.calibration_step2()
        torch.cuda.synchronize()
    return run


def main():
    layers = sys.argv[1:] or ["fc1", "qkv"]
    with tempfile.TemporaryDirectory(prefix="p4v_phases_") as tmp:
        _lib.LIB_PATH = build_phase_lib(tmp)
        L = _lib.lib()
        L.p4v_sweep_phase_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
        buf = (C.c_ulonglong * (6 * N_PHASES))()
        for kind in layers:
            run = layer_runner(kind)
            run()
            _lib.check(L.p4v_sweep_phase_clocks(buf, 1), "p4v_sweep_phase_clocks")   # reset after the warm-up
            run()
            _lib.check(L.p4v_sweep_phase_clocks(buf, 1), "p4v_sweep_phase_clocks")
            print(f"== {kind} (one search round, n_H = 24, eq_n = 100)")
            for k, name in enumerate(KINDS):
                t = buf[k * N_PHASES:(k + 1) * N_PHASES]
                if t[6] == 0:
                    continue
                shares = ", ".join(f"{p} {100.0 * t[i] / t[6]:.1f}%" for i, p in enumerate(CONSUMER))
                other = 100.0 * (t[6] - sum(t[:6])) / t[6]
                print(f"  {name:12s} consumer {t[6] / 1e9:.3f} Gcycles: {shares}, other (issue, tables, loads) {other:.1f}%")
                if t[8]:
                    print(f"  {'':12s} producer {t[8] / 1e9:.3f} Gcycles: wait empty {100.0 * t[7] / t[8]:.1f}%")


if __name__ == "__main__":
    main()
