"""The torch-op voxel-grid ports of tests/autograd_voxel_ports.py against the real reference's outputs and gradients
(tests/golden/autograd_voxel.npz, tests/golden/make_golden_autograd_voxel.py); needs no GPU.  The ports are the
gradient oracle of tests/test_gpu_voxel_autograd.py."""
import numpy as np
import pytest

import autograd_voxel_ports as P
from autograd_voxel_cases import CASES, run, scene
from conftest import assert_close_to_max, golden

PORT = (P.events_to_voxel_torch, P.events_to_neg_pos_voxel_torch)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_port_values_and_gradients(case):
    g = golden("autograd_voxel")
    name = case["name"]
    inputs = scene(case)
    for k, v in inputs.items():
        assert np.array_equal(v.numpy(), g["%s/in_%s" % (name, k)], equal_nan=True), "%s: scene %s changed" % (name, k)
    outs, weights, grads = run(case, PORT, inputs)
    for i, (o, w) in enumerate(zip(outs, weights)):
        assert np.array_equal(w.numpy(), g["%s/w%d" % (name, i)])
        assert_close_to_max(o.numpy(), g["%s/out%d" % (name, i)], 1e-6, "%s out%d" % (name, i))
    for k in ("ts", "ps"):
        ref = g["%s/grad_%s" % (name, k)]
        if ref.size == 0:
            assert grads[k] is None, "%s: the reference leaves %s without a gradient" % (name, k)
        else:
            assert grads[k] is not None, "%s: no gradient for %s" % (name, k)
            assert_close_to_max(grads[k].numpy(), ref, 1e-5, "%s grad %s" % (name, k))
