"""Host-side mirror of the reference's `examples/seismic` callers of the hot path."""
from .model import SeismicModel, Model, demo_model, initialize_damp, damp_profile  # noqa: F401
from .source import (TimeAxis, PointSource, Receiver, Shot, WaveletSource, RickerSource,  # noqa: F401
                     GaborSource)
from .geometry import AcquisitionGeometry, setup_geometry, setup_rec_coords  # noqa: F401
from .acoustic import AcousticWaveSolver, iso_stencil  # noqa: F401
from .acoustic import ForwardOperator as AcousticForwardOperator  # noqa: F401
from .acoustic import AdjointOperator as AcousticAdjointOperator  # noqa: F401
from .tti import AnisotropicWaveSolver, kernel_centered  # noqa: F401
from .tti import ForwardOperator as TTIForwardOperator  # noqa: F401
from .self_adjoint import (SaIsoAcousticWaveSolver, IsoFwdOperator, IsoAdjOperator, setup_w_over_q,  # noqa: F401
                           acoustic_sa_setup)
from .self_adjoint import iso_stencil as sa_iso_stencil  # noqa: F401
from .viscoacoustic import ViscoacousticWaveSolver  # noqa: F401
