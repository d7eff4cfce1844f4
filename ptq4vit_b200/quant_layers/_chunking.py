"""Memory-bounded searches: how many chunks a layer's search workspace is split into.

The search of a layer needs operand images of every candidate for all of its rows (Linear) or images (MatMul).  When
that workspace does not fit in the device memory that is free, the library searches one chunk of rows / images at a
time and adds the chunks' scores (the reference's `calib_need_batching`, quant_layers/linear.py:365-378,
matmul.py:396-409).  The captured tensors stay whole; only the workspace is sized for one chunk.
"""
import os

import torch

# Device memory kept free besides the workspace: the CUDA context's own allocations and the small tensors of the call
# (step sizes, score log) must still fit next to it.
SAFETY_MARGIN_BYTES = 512 << 20
BUDGET_ENV = "P4V_WORKSPACE_BUDGET"


def device_free_bytes(device):
    """The free device memory plus what torch's caching allocator holds without handing it out, minus
    SAFETY_MARGIN_BYTES."""
    free, _ = torch.cuda.mem_get_info(device)
    idle = torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)
    return free + idle - SAFETY_MARGIN_BYTES


def workspace_budget(device):
    """Bytes a search workspace may take on `device`: P4V_WORKSPACE_BUDGET if set, else device_free_bytes."""
    env = os.environ.get(BUDGET_ENV)
    if env:
        return int(env)
    return device_free_bytes(device)


def choose_chunks(n, granule, workspace_bytes, budget):
    """Smallest number of chunks of a layer of `n` units (rows or images) whose search workspace fits in `budget`.

    Every chunk but the last holds a multiple of `granule` units.  `workspace_bytes(per_chunk)` is the workspace the
    library plans for chunks of `per_chunk` units, with 0 meaning the whole layer at once.  Returns
    (per_chunk, n_chunks); per_chunk == 0 (one chunk) when the whole layer fits.  Raises MemoryError when even a
    chunk of `granule` units does not fit."""
    if workspace_bytes(0) <= budget:
        return 0, 1
    for k in range(2, -(-n // granule) + 1):
        per = -(-(-(-n // k)) // granule) * granule      # ceil(n / k) rounded up to the granule
        if per >= n:
            continue
        if workspace_bytes(per) <= budget:
            return per, -(-n // per)
    smallest = workspace_bytes(min(granule, n)) if granule < n else workspace_bytes(0)
    raise MemoryError(f"search workspace does not fit: one chunk of {min(granule, n)} of {n} units needs {smallest} bytes, "
                      f"the budget is {budget} bytes (free device memory minus {SAFETY_MARGIN_BYTES} bytes, or ${BUDGET_ENV})")
