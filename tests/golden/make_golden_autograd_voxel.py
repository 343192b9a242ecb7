"""Generate the voxel-grid gradients of the UNMODIFIED reference (TimoStoff/event_utils, loaded through
oracle/ref_loader.py) behind tests/test_autograd_voxel_port.py:

    EVK_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden_autograd_voxel.py

Each case of tests/autograd_voxel_cases.py stores its inputs, the reference's outputs, the weights R of the loss
sum(out * R) and the gradients autograd gives ts and ps (ps of the neg/pos split gets none: stored as an empty
array).  Runs on the CPU, the only device the reference's voxel grids run on; autograd_voxel.npz stays under 1 MB.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from autograd_voxel_cases import CASES, run, scene  # noqa: E402
from oracle import ref_loader  # noqa: E402

ref = ref_loader.load()
torch.set_num_threads(1)

fns = (ref.voxel_grid.events_to_voxel_torch, ref.voxel_grid.events_to_neg_pos_voxel_torch)
out = {}
for case in CASES:
    inputs = scene(case)
    outs, weights, grads = run(case, fns, inputs)
    res = {"in_" + k: v.numpy() for k, v in inputs.items()}
    for i, (o, w) in enumerate(zip(outs, weights)):
        res["out%d" % i], res["w%d" % i] = o.numpy(), w.numpy()
    for k, g in grads.items():
        res["grad_" + k] = np.zeros(0, np.float32) if g is None else g.numpy()
    for k, v in res.items():
        out["%s/%s" % (case["name"], k)] = v

path = os.path.join(HERE, "autograd_voxel.npz")
np.savez_compressed(path, **out)
print("autograd_voxel.npz %.1f KB" % (os.path.getsize(path) / 1024))
