"""nonlinearsolve.jl_b200 — H100-native Newton iteration core behind the NonlinearSolve.jl first-order solver API.

Only what the hot path needs lives here: `csrc/` (hand-written sm_90a CUDA + the C ABI of include/b200newton.h),
`_abi.py` (ctypes binding) and `api.py` (host-side mirror of the reference interface).  Import through the root shim
`nonlinearsolve_jl_b200` (the directory name contains a dot, as the task layout asks).
"""
from . import _abi as abi  # noqa: F401
from .api import *  # noqa: F401,F403
from .api import (Context, DeviceVector, default_context, device_count, ReturnCode, successful_retcode, NLStats, NonlinearSolution,  # noqa: F401
                  Brusselator2D, Brusselator3D, QuadraticFunction, TridiagQuadFunction, NonlinearFunction, TracerSparsityDetector,
                  NonlinearProblem, remake, KrylovJL_GMRES, LUFactorization, AutoForwardDiff, AutoFiniteDiff, EisenstatWalkerForcing2, BackTracking, BlockJacobi, PseudoTransient, RadiusUpdateSchemes,
                  AbsNormSafeBestTerminationMode, AbsNormSafeTerminationMode, AbsNormTerminationMode, NormTerminationMode, RelTerminationMode, RelNormTerminationMode,
                  AbsTerminationMode, RelNormSafeTerminationMode, RelNormSafeBestTerminationMode, Multigrid, LevenbergMarquardt, Broyden, LimitedMemoryBroyden, Klement, KLUFactorization, UMFPACKFactorization, SparseBandLU, ILU0, SparseILU0, RugeStubenAMG, SmoothedAggregationAMG, SparseAMG, amg_split, NewtonRaphson, TrustRegion,
                  SparseJacobian, JacobianOperator, GmresSolver, NonlinearSolveCache, init, step_b, solve_b, reinit_b, EnsembleProblem,
                  EnsembleB200, EnsembleSolution, EnsembleCache, Communicator, shard_range, coloring_column, solve, _DeviceProblem)
