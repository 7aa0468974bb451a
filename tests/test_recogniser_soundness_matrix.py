"""Every (case, mutation) the recogniser accepts, run for K steps on the GPU against its float64 twin (the same
builder at float64, which must run on the interpreter): every slot of every field, halo included, and every
sparse function (traces, `srca`), plus `grad` and the snapshots where present. Tolerances are the north-star
ones of BASELINE.json: rel L-inf 1e-5 for the isotropic and self-adjoint updates, 1e-4 for TTI."""
import numpy as np
import pytest

import recogniser_cases as RC
from test_recogniser_soundness import ACCEPTED

pytestmark = pytest.mark.gpu

TOL = {'iso': 1e-5, 'sa': 1e-5, 'tti': 1e-4}


def _lib():
    from devito_b200 import _lib as L_
    return L_.lib()


def _arrays(b):
    out = {}
    for n, f in b.functions.items():
        out[n] = np.array(f.data if getattr(f, 'is_SparseFunction', False) else f.data_with_halo, dtype=np.float64)
    return out


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


@pytest.mark.parametrize('case,mutation', sorted(ACCEPTED), ids=[f'{c}-{m}' for c, m in sorted(ACCEPTED)])
def test_accepted_matches_float64(case, mutation):
    gpu = RC.build(case, mutation)
    assert gpu.op.backend == 'cuda-sm90a'
    before = _arrays(gpu)
    launches = _lib().b2_launch_count()
    gpu.op.apply(**gpu.kwargs)
    assert _lib().b2_launch_count() > launches and _lib().b2_last_sweep_kernel().decode(), "no kernel ran"
    got = _arrays(gpu)
    twin = RC.build(case, mutation, np.float64)
    assert twin.op.backend == 'numpy-interpreter'
    assert set(twin.functions) == set(gpu.functions)
    twin.op.apply(**twin.kwargs)
    want = _arrays(twin)
    tol = TOL[gpu.family]
    written = 0
    for n in sorted(want):
        assert _rel(got[n], want[n]) < tol, (n, _rel(got[n], want[n]))
        written += not np.array_equal(before[n], want[n])
    assert written, "the float64 twin wrote nothing"
