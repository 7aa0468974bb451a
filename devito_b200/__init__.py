"""devito_b200 — an H100-native execution backend behind the Devito `Operator` API for the
explicit time-stepping hot path of acoustic / TTI wave propagation.

Public names follow the reference package (`from devito import ...`, SURVEY Appendix B) so
that scripts written against it keep working for the supported path.
"""
from .parameters import configuration, switchconfig  # noqa: F401
from .logger import info, warning, error, perf, debug, set_log_level  # noqa: F401
from .exceptions import (InvalidArgument, InvalidOperator, ExecutionError,  # noqa: F401
                         BackendUnavailable, DevitoError)
from .symbolics import (sin, cos, sqrt, Abs, sign, exp, floor, INT, Derivative,  # noqa: F401
                        retrieve_functions, retrieve_derivatives, div, grad)
from .types import (Grid, SubDomain, Dimension, SpaceDimension, TimeDimension,  # noqa: F401
                    SteppingDimension, SubDimension, DefaultDimension, ConditionalDimension,
                    Function, TimeFunction, Constant, Buffer, NODE, CELL)
from .sparse import SparseFunction, SparseTimeFunction, Injection, Interpolation  # noqa: F401
from .equation import Eq, Inc, FreeSurface, solve  # noqa: F401
from .operator import Operator, PerformanceSummary  # noqa: F401
from .builtins import (norm, sumall, inner, mmin, mmax, assign, smooth, gaussian_smooth,  # noqa: F401
                       initialize_function)
from .distributed import init_distributed  # noqa: F401

__version__ = '0.1.0'


class _OutOfScope:
    """Names the reference's examples import at module level but that belong to SURVEY §8f
    ("next") or out-of-scope rows: importing works, using raises."""
    _what = ''

    def __init__(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__} is outside this backend's scope: {self._what}")


class CheckpointOperator(_OutOfScope):
    _what = "the pyrevolve adapters (devito/checkpointing/checkpoint.py) are not provided; the checkpointed " \
            "acoustic gradient is `AcousticWaveSolver.jacobian_adjoint(rec, checkpointing=True, n_checkpoints=...)`, " \
            "which runs its binomial schedule (devito_b200.revolve) inside one library call"


class DevitoCheckpoint(_OutOfScope):
    _what = CheckpointOperator._what


class Revolver(_OutOfScope):
    _what = CheckpointOperator._what


def install_as_devito():
    """Expose this package under the import name `devito` (and its `devito.types`,
    `devito.builtins`, `devito.tools`, `devito.symbolics`, `devito.logger` sub-modules) so that
    unmodified user scripts — e.g. the reference's `examples/seismic` — import it."""
    import sys
    import types as _t
    from . import builtins as _b, tools as _tools, symbolics as _s, logger as _l, sparse as _sp
    from . import types as _ty
    me = sys.modules[__name__]
    sys.modules['devito'] = me
    sys.modules['devito.builtins'] = _b
    sys.modules['devito.tools'] = _tools
    sys.modules['devito.symbolics'] = _s
    sys.modules['devito.logger'] = _l
    tmod = _t.ModuleType('devito.types')
    for src in (_ty, _sp):
        for k in dir(src):
            if not k.startswith('__'):
                setattr(tmod, k, getattr(src, k))
    sys.modules['devito.types'] = tmod
    sys.modules['devito.types.sparse'] = _sp
    me.types = tmod
    return me
