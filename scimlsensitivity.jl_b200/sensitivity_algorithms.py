"""Sensitivity-algorithm and VJP-choice structs: the `sensealg=` / `autojacvec=` plugin surface.

Mirrors /root/reference/src/sensitivity_algorithms.jl: BacksolveAdjoint :254-278, InterpolatingAdjoint :378-405,
QuadratureAdjoint :486-510, GaussAdjoint :591-611, VJPChoice family :1426-1602 and the traits :1606-1733.
Field names, keyword names and defaults are the reference's; the only addition is `B200VJP`, the
hand-differentiated device VJP that this engine uses for the named RHS families (it plays the role a
`VJPChoice` back-end plays in src/derivative_wrappers.jl:256-267), and the `B200Adjoint` wrapper that selects
the device path in `_concrete_solve_adjoint` (the extension pattern of ext/SciMLSensitivityMooncakeExt.jl:123-240).
"""
from dataclasses import dataclass, replace
from typing import Any, Optional


# ---- VJP choices (src/sensitivity_algorithms.jl:1426-1602) ----
class VJPChoice:
    pass


@dataclass(frozen=True)
class ZygoteVJP(VJPChoice):
    allow_nothing: bool = False


@dataclass(frozen=True)
class EnzymeVJP(VJPChoice):
    chunksize: int = 0


@dataclass(frozen=True)
class TrackerVJP(VJPChoice):
    allow_nothing: bool = False


@dataclass(frozen=True)
class ReverseDiffVJP(VJPChoice):
    compile: bool = False


@dataclass(frozen=True)
class MooncakeVJP(VJPChoice):
    pass


@dataclass(frozen=True)
class ReactantVJP(VJPChoice):
    allow_scalar: bool = False


@dataclass(frozen=True)
class B200VJP(VJPChoice):
    """Hand-differentiated sm_90a device VJP for a named RHS family (csrc/families.cuh)."""
    pass


# ---- adjoint sensitivity algorithms ----
class AbstractAdjointSensitivityAlgorithm:
    chunk_size: int
    autodiff: bool
    diff_type: str


@dataclass(frozen=True)
class BacksolveAdjoint(AbstractAdjointSensitivityAlgorithm):
    chunk_size: int = 0
    autodiff: bool = True
    diff_type: str = "central"
    autojacvec: Any = None
    checkpointing: bool = True
    noisemixing: bool = False


@dataclass(frozen=True)
class InterpolatingAdjoint(AbstractAdjointSensitivityAlgorithm):
    chunk_size: int = 0
    autodiff: bool = True
    diff_type: str = "central"
    autojacvec: Any = None
    checkpointing: bool = False
    noisemixing: bool = False


@dataclass(frozen=True)
class QuadratureAdjoint(AbstractAdjointSensitivityAlgorithm):
    chunk_size: int = 0
    autodiff: bool = True
    diff_type: str = "central"
    autojacvec: Any = None
    abstol: float = 1.0e-6
    reltol: float = 1.0e-3
    diff_tunables: bool = True


@dataclass(frozen=True)
class GaussAdjoint(AbstractAdjointSensitivityAlgorithm):
    chunk_size: int = 0
    autodiff: bool = True
    diff_type: str = "central"
    autojacvec: Any = None
    checkpointing: bool = False
    diff_tunables: bool = True


@dataclass(frozen=True)
class GaussKronrodAdjoint(AbstractAdjointSensitivityAlgorithm):
    """src/sensitivity_algorithms.jl:689-703: GaussAdjoint with an error-controlled Gauss-Kronrod quadrature of every
    accepted reverse step (IntegratingGKSumCallback, src/gauss_adjoint.jl:820-825).  Device: adaptive steppers."""
    chunk_size: int = 0
    autodiff: bool = True
    diff_type: str = "central"
    autojacvec: Any = None
    checkpointing: bool = False


@dataclass(frozen=True)
class B200Adjoint(AbstractAdjointSensitivityAlgorithm):
    """`sensealg=B200Adjoint(GaussAdjoint())`: run `inner` on the B200 engine (SURVEY.md 8b)."""
    inner: Any = None
    block_threads: int = 0
    stored_noise: bool = False
    checkpoint_every: int = 1     # fixed-step Tsit5 with inner.checkpointing: keep the forward state every C steps and re-solve
                                  # each segment in the reverse pass (the reference's `checkpoints` grid, src/interpolating_adjoint.jl:54-112)

    def __post_init__(self):
        if self.inner is None:
            object.__setattr__(self, "inner", InterpolatingAdjoint())
        if not isinstance(self.inner, (BacksolveAdjoint, InterpolatingAdjoint, QuadratureAdjoint, GaussAdjoint, GaussKronrodAdjoint)):
            raise TypeError("B200Adjoint wraps one of the continuous adjoints")


def setvjp(sensealg, vjp):
    """src/sensitivity_algorithms.jl:272-278 and twins."""
    if isinstance(sensealg, B200Adjoint):
        return replace(sensealg, inner=replace(sensealg.inner, autojacvec=vjp))
    return replace(sensealg, autojacvec=vjp)


# ---- traits (src/sensitivity_algorithms.jl:1606-1733) ----
def alg_autodiff(alg):
    return alg.autodiff


def get_chunksize(alg):
    return alg.chunk_size


def diff_type(alg):
    return alg.diff_type


def get_jacvec(alg):
    return alg.autojacvec if isinstance(alg.autojacvec, bool) else True


def needs_checkpointing(alg, sol):
    if getattr(sol.prob, "is_sde", False):
        return alg.checkpointing
    return alg.checkpointing or not sol.dense


def ischeckpointing(alg, sol=None):
    if isinstance(alg, B200Adjoint):
        alg = alg.inner
    if isinstance(alg, BacksolveAdjoint):
        return alg.checkpointing
    if isinstance(alg, (InterpolatingAdjoint, GaussAdjoint, GaussKronrodAdjoint)):
        return alg.checkpointing if sol is None else needs_checkpointing(alg, sol)
    return False


def isnoisemixing(alg):
    if isinstance(alg, B200Adjoint):
        alg = alg.inner
    return bool(getattr(alg, "noisemixing", False))


def supports_functor_params(alg):
    return isinstance(alg, (GaussAdjoint, GaussKronrodAdjoint))      # AbstractGAdjoint (src/sensitivity_algorithms.jl:712, :1692-1699)


def supports_structured_vjp(vjp):
    return isinstance(vjp, (ZygoteVJP, EnzymeVJP, MooncakeVJP, ReactantVJP))


SENSEALG_CODE = {InterpolatingAdjoint: "interpolating", GaussAdjoint: "gauss", QuadratureAdjoint: "quadrature",
                 BacksolveAdjoint: "backsolve", GaussKronrodAdjoint: "gauss_kronrod"}


def sensealg_name(alg):
    if isinstance(alg, B200Adjoint):
        alg = alg.inner
    return SENSEALG_CODE[type(alg)]
