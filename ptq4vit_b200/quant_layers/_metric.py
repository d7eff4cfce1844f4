"""Per-element weight of the search metric, as the search kernels take it.

The kernels score a candidate as -(g * (y - yhat))^2 averaged the reference's way, g being the cached
gradient of the Hessian metric (quant_layers/linear.py:417-420, matmul.py:473-477, conv.py:517-520).  The
reference's other squared-error metrics are the same expression with another per-element weight:

  L2_norm                   -(y - yhat)^2                 g = 1            (linear.py:411-412)
  linear_weighted_L2_norm   -|y| (y - yhat)^2             g = sqrt(|y|)    (linear.py:413-414)
  square_weighted_L2_norm   -(y (y - yhat))^2             g = y            (linear.py:415-416)

`cosine` and `L1_norm` are not weighted squared errors and are not implemented here; `pearson` is broken
in the reference itself (linear.py:433).
"""
import torch


METRICS = ("hessian", "L2_norm", "linear_weighted_L2_norm", "square_weighted_L2_norm")


def check_metric(metric):
    """Raise, as metric_weight would, for a metric the search kernels do not implement -- before any work is done."""
    if metric not in METRICS:
        raise NotImplementedError(f"metric {metric} not implemented!")


def metric_weight(metric, y, raw_grad, what):
    if metric == "hessian":
        assert raw_grad is not None, f"raw_grad is None in {what}!"
        return raw_grad
    if metric == "L2_norm":
        return torch.ones_like(y)
    if metric == "linear_weighted_L2_norm":
        return y.abs().sqrt_()
    if metric == "square_weighted_L2_norm":
        return y
    raise NotImplementedError(f"metric {metric} not implemented!")
