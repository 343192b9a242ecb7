"""Adversarial small cases: the oracle must agree with the real reference on results AND on error behaviour.  The
reference's results (or the fact that it raised) were stored by tests/golden/make_golden_random.py."""
import numpy as np

from conftest import assert_close_to_max, golden
from edge_cases import cases


def _run(fn):
    try:
        return fn(), None
    except (IndexError, ValueError, RuntimeError) as e:
        return None, type(e)


def test_oracle_matches_reference_on_edge_cases(oracle, capsys):
    g = golden("edge_cases")
    values, raised, lengths = g["values"], g["raised"], g["lengths"]
    offsets = np.concatenate(([0], np.cumsum(lengths)))
    assert len(raised) == 3 * 300
    slot = 0

    def check(o, oe, what):
        nonlocal slot
        re = bool(raised[slot])
        r = values[offsets[slot]:offsets[slot + 1]]
        slot += 1
        assert re == (oe is not None), (what, re, oe)
        if not re:
            assert_close_to_max(np.asarray(o).ravel(), r, 1e-6 if what[0] == "voxel" else 2e-6, "%s case %d %s" % what)
            return 1, 0
        return 0, 1

    checked = errors = 0
    for c in cases(2024, 300):
        hw = (c["H"], c["W"])
        o, oe = _run(lambda: oracle.voxel_f32(c["x"], c["y"], c["t"], c["p"], c["B"], hw))
        a, b = check(o, oe, ("voxel", c["k"], None))
        checked, errors = checked + a, errors + b
        for interp in (None, "bilinear"):
            kw = dict(sensor_size=hw, clip_out_of_range=c["clip"], interpolation=interp, padding=c["padding"])
            o, oe = _run(lambda: oracle.image_torch_f32(c["x"], c["y"], c["p"], **kw))
            a, b = check(o, oe, ("image", c["k"], interp))
            checked, errors = checked + a, errors + b
    capsys.readouterr()
    assert checked > 300 and errors > 50     # both regimes are exercised
