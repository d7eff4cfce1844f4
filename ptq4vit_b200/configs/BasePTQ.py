"""Operator factory with the reference's BasePTQ contract (configs/BasePTQ.py:1-62): module-level kwargs dicts that
experiment code mutates in place, and get_module(module_type, *args).

BasePTQ is the baseline of the reference's experiment matrix (example/test_all.py:18-119): the patch embedding gets ONE
weight step size (BatchingEasyQuantConv2d, layer-wise EasyQuant, activations left in FP32); every Linear and MatMul is
the plain Batching class with one block (no post-GELU twin-uniform fc2, no split-of-softmax matmul2), one search round,
candidates from eq_alpha 0.5 to eq_beta 1.2.

The dicts keep the reference's default `metric = "cosine"`, verbatim.  The search kernels implement the Hessian and the
squared-error metrics only, so with that default every module's `calibration_step2()` raises NotImplementedError naming
the metric, before any kernel is launched.  The reference's experiments run BasePTQ with `metric = "hessian"` (the
`cfg_modifier` of example/test_all.py:53-78), which is what runs here:

    from ptq4vit_b200.configs import BasePTQ as cfg
    for d in (cfg.ptqsl_conv2d_kwargs, cfg.ptqsl_linear_kwargs, cfg.ptqsl_matmul_kwargs):
        d["metric"] = "hessian"
"""
from ..quant_layers.conv import BatchingEasyQuantConv2d
from ..quant_layers.linear import PTQSLBatchingQuantLinear
from ..quant_layers.matmul import PTQSLBatchingQuantMatMul

bit = 8
conv_fc_name_list = ["qconv", "qlinear_qkv", "qlinear_proj", "qlinear_MLP_1", "qlinear_MLP_2", "qlinear_classifier", "qlinear_reduction"]
matmul_name_list = ["qmatmul_qk", "qmatmul_scorev"]
w_bit = {name: bit for name in conv_fc_name_list}
a_bit = {name: bit for name in conv_fc_name_list}
A_bit = {name: bit for name in matmul_name_list}
B_bit = {name: bit for name in matmul_name_list}

ptqsl_conv2d_kwargs = {"metric": "cosine", "eq_alpha": 0.5, "eq_beta": 1.2, "eq_n": 100, "search_round": 1, "n_V": 1, "n_H": 1}
ptqsl_linear_kwargs = {"metric": "cosine", "eq_alpha": 0.5, "eq_beta": 1.2, "eq_n": 100, "search_round": 1,
                       "n_V": 1, "n_H": 1, "n_a": 1}
ptqsl_matmul_kwargs = {"metric": "cosine", "eq_alpha": 0.5, "eq_beta": 1.2, "eq_n": 100, "search_round": 1,
                       "n_G_A": 1, "n_V_A": 1, "n_H_A": 1, "n_G_B": 1, "n_V_B": 1, "n_H_B": 1}


def get_module(module_type, *args, **kwargs):
    """reference: configs/BasePTQ.py:47-62.  The kwargs dicts are read at call time, so an experiment's cfg_modifier can
    edit them between calls (example/test_all.py:53-78).  q, k and v each get their own row blocks; unlike PTQ4ViT the
    classifier head keeps the shared n_V."""
    if module_type == "qconv":
        opts = {**kwargs, **ptqsl_conv2d_kwargs}
        return BatchingEasyQuantConv2d(*args, **opts, w_bit=w_bit["qconv"], a_bit=32)   # activation quantizer off
    if "qlinear" in module_type:
        opts = {**kwargs, **ptqsl_linear_kwargs}
        if module_type == "qlinear_qkv":
            opts["n_V"] *= 3
        return PTQSLBatchingQuantLinear(*args, **opts, w_bit=w_bit[module_type], a_bit=a_bit[module_type])
    if "qmatmul" in module_type:
        opts = {**kwargs, **ptqsl_matmul_kwargs}
        return PTQSLBatchingQuantMatMul(*args, **opts, A_bit=A_bit[module_type], B_bit=B_bit[module_type])
    raise NotImplementedError(f"unknown module type {module_type}")
