"""Generate the gradients of the UNMODIFIED reference (TimoStoff/event_utils, loaded through oracle/ref_loader.py)
behind tests/test_autograd_port.py:

    EVK_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden_autograd.py

Each case stores its inputs, the reference's forward outputs, the weights of the loss sum(out * R) and the
gradients autograd gives every input that requires grad.  An input the reference leaves without a gradient is
stored as an empty array under its gradient's key.  Runs on the CPU; autograd.npz stays well under 1 MB.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from autograd_cases import CASES, run, scene  # noqa: E402
from oracle import ref_loader  # noqa: E402

ref = ref_loader.load()
torch.set_num_threads(1)


fns = (ref.image.events_to_image_torch, ref.image.events_to_timestamp_image_torch,
       ref.optic_flow.warp_events_flow_torch)
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

path = os.path.join(HERE, "autograd.npz")
np.savez_compressed(path, **out)
print("autograd.npz %.1f KB" % (os.path.getsize(path) / 1024))
