"""scimlsensitivity.jl_b200 -- H100-native (Hopper) ensemble continuous-adjoint engine.

One hot path of SciML/SciMLSensitivity.jl (reverse-mode continuous adjoints over an EnsembleProblem) rebuilt as
hand-written sm_90a CUDA kernels behind a C ABI (include/b200adj.h), with this thin host layer mirroring the
reference's `sensealg=` plugin surface.  Import as `scimlsensitivity_jl_b200` (the directory name carries a dot).
"""
from . import _lib
from . import distributed
from ._lib import B200AdjError, build
from .concrete_solve import (ChainRulesOriginator, NoTangent, ReverseDiffOriginator, TrackerOriginator,
                             _concrete_solve_adjoint, clear_handle_cache, solve)
from .distributed import allreduce_dp, shard_bounds
from .engine import DeviceEnsemble
from .family_plugin import build_family_plugin, register_family
from .problems import (EM, AdjointSensitivityParameterCompatibilityError, AffineAffect, AffineCost, ContinuousCallback, VectorContinuousCallback, PresetTimeCallback, EnsembleB200, EnsembleProblem,
                       EnsembleSolution, EulerHeun, FAMILIES, ODEProblem, ParamAffine, QuadraticRunningCost, Rosenbrock23, SDEProblem, Tsit5)
from .sensitivity_algorithms import (B200Adjoint, B200VJP, BacksolveAdjoint, EnzymeVJP, GaussAdjoint, GaussKronrodAdjoint,
                                     InterpolatingAdjoint, MooncakeVJP, QuadratureAdjoint, ReactantVJP,
                                     ReverseDiffVJP, TrackerVJP, VJPChoice, ZygoteVJP, alg_autodiff, diff_type,
                                     get_chunksize, get_jacvec, ischeckpointing, isnoisemixing, sensealg_name, setvjp,
                                     supports_functor_params, supports_structured_vjp)
from .sensitivity_interface import adjoint_sensitivities

__all__ = [n for n in dir() if not n.startswith("_")] + ["_concrete_solve_adjoint"]
