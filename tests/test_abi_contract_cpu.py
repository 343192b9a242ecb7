"""No-GPU half of the ABI contract tests: every declared entry has a contract case or a stated reason not to, and the
workspace query of every batched loss returns 0 exactly for the arguments its entries refuse.  The GPU half is
tests/test_gpu_abi_contract.py."""
import ctypes

import pytest
import torch

import abi_contract_cases as C
from test_abi import declared_symbols

E_ARG, E_WORKSPACE = -1, -3
PLACEHOLDER = 1 << 20          # a non-null, 256-byte aligned pointer that is never dereferenced


def _lib():
    from event_utils_b200 import _lib
    return _lib.load()


def test_every_declared_entry_has_a_case_or_a_reason():
    P = C.protos()
    covered = set(C.batched_entries()) | set(C.SIMPLE)
    excluded = C.EXCLUDED
    queries = {s for s in P if s.endswith("_workspace_bytes")}
    for name in declared_symbols():
        if name in queries:
            continue
        assert (name in covered) != (name in excluded), "%s: needs a contract case or a reason to have none (not both)" % name
    for name, reason in excluded.items():
        assert name in P and len(reason) > 10, name
    # every query sizes at least one covered entry
    used = {C.workspace_query(e) for e in covered} - {None}
    assert queries == used, queries - used


def test_the_case_table_builds():
    cases = C.batched_cases() + C.simple_cases()
    assert {c.entry for c in cases} == set(C.batched_entries()) | set(C.SIMPLE)
    P = C.protos()
    for c in cases:
        names = set(P[c.entry])
        missing = names - set(c.values) - {"workspace", "workspace_bytes", "stream"}
        assert not missing, (c.id, missing)
        assert c.compared(), c.id
        for o in c.outputs():
            assert o in names, (c.id, o)
        c.workspace_bytes(_lib())


def _call(L, entry, v, ws, ws_bytes):
    args = []
    for name in C.protos()[entry]:
        if name == "workspace":
            args.append(ws)
        elif name == "workspace_bytes":
            args.append(ws_bytes)
        elif name == "stream":
            args.append(None)
        elif name in v:
            args.append(v[name])
        else:
            args.append(PLACEHOLDER)      # every array of the call
    return getattr(L, entry)(*args)


@pytest.mark.parametrize("entry", C.batched_entries())
def test_query_returns_zero_exactly_where_the_entry_refuses(entry):
    """At each limit and one past it (batch, batch J and batch M, J and M, the node grid against the sensor and its
    node counts, the 2^30-pixel canvas, products that wrap an int): a refused call gets EVK_E_ARG and its query 0; an
    accepted shape gets a non-zero query (0 only at batch 0, which needs no workspace), and the entry refuses one byte
    less and a workspace 128 bytes off its alignment with EVK_E_WORKSPACE.  Placeholder pointers: no call here may
    reach a device, so the test runs only where none is visible."""
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is visible: an accepted call would launch on placeholder pointers "
                    "(tests/test_gpu_abi_contract.py covers the accepted side there)")
    L = _lib()
    q = C.workspace_query(entry)
    bad = []
    for label, over, accepted in C.limit_points(entry):
        v = C.sweep_values(entry, over)
        nbytes = getattr(L, q)(*C.query_args(q, v))
        if not accepted:
            rc = _call(L, entry, v, PLACEHOLDER, 1 << 62)
            if nbytes != 0 or rc != E_ARG:
                bad.append("%s: refused shape, query %d, entry rc %d" % (label, nbytes, rc))
            continue
        if v["batch"] == 0:
            rc = _call(L, entry, v, PLACEHOLDER, 0)
            if nbytes != 0 or rc != 0:
                bad.append("%s: query %d, entry rc %d" % (label, nbytes, rc))
            continue
        if nbytes == 0 or nbytes % 256:
            bad.append("%s: accepted shape, query %d" % (label, nbytes))
            continue
        rc_short = _call(L, entry, v, PLACEHOLDER, nbytes - 1)
        rc_off = _call(L, entry, v, PLACEHOLDER + 128, nbytes)
        if rc_short != E_WORKSPACE or rc_off != E_WORKSPACE:
            bad.append("%s: query %d, one byte short rc %d, misaligned rc %d" % (label, nbytes, rc_short, rc_off))
    assert not bad, "%s:\n  %s" % (entry, "\n  ".join(bad))


def test_the_queries_of_the_reported_shapes_return_zero():
    """the four shapes at which the queries once returned hundreds of MB to 70 GB for calls their entries refuse"""
    L = _lib()
    assert L.evk_cmax_motion_candidates_workspace_bytes(65536, 1, 10, 10) == 0
    assert L.evk_cmax_motion_segment_workspace_bytes(16384, 4, 10, 10) == 0
    assert L.evk_motion_timestamp_candidates_workspace_bytes(1024, 32, 10, 10) == 0
    assert L.evk_cmax_motion_objective_workspace_bytes(1, 40000, 40000) == 0
    # and their neighbours inside the limits are not 0
    assert L.evk_cmax_motion_candidates_workspace_bytes(65535, 1, 10, 10) > 0
    assert L.evk_cmax_motion_segment_workspace_bytes(16383, 4, 10, 10) > 0
    assert L.evk_motion_timestamp_candidates_workspace_bytes(1023, 32, 10, 10) > 0
    assert L.evk_cmax_motion_objective_workspace_bytes(1, 32767, 32767) > 0

