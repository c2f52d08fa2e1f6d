"""krylovkit.jl_b200 — H100-native Krylov inner-loop engine behind KrylovKit.jl's API.

The directory name contains a dot, so import it through the top-level alias module:

    import krylovkit_jl_b200 as kk

Everything numerical runs in libb200krylov.so (hand-written sm_90a CUDA, C-ABI declared
in include/b200krylov.h).  Importing the package does not need a GPU; creating a
B200Context does, and fails loudly without one (no CPU fallback).
"""
from . import _lib
from ._lib import B200Error, DimensionMismatch, LibraryMissing
from .algorithms import (Arnoldi, BiArnoldi, BiCGStab, BlockLanczos, CG, ClassicalGramSchmidt, ClassicalGramSchmidt2,
                         ClassicalGramSchmidtIR, ConvergenceInfo, GKL, GMRES, GolubYe, KrylovDefaults,
                         Lanczos, LSMR, MINRES, ModifiedGramSchmidt, ModifiedGramSchmidt2,
                         ModifiedGramSchmidt2Blocked, ModifiedGramSchmidtIR, Orthogonalizer, cgs, cgs2, cgsr, mgs,
                         mgs2, mgs2b, mgsr)
from .operators import (B200CSR, B200Dense, B200Operator, B200Pencil, apply, apply_adjoint, apply_normal,
                        apply_normal_gram, genapply)
from .orthonormal import (OrthonormalBasis, basistransform_, cross_inner, orthogonalize_, orthonormalize_,
                          project_, rank1update_, rmul_givens_, rmul_householder_, unproject_)
from .vectors import B200Context, B200Vec, cache_release, inner, norm

__all__ = [n for n in dir() if not n.startswith("_")]
from .dense import EigSorter
from .eigsolve import eigselector, eigsolve
from .linsolve import linselector, linsolve
from .schursolve import ComplexVec, realeigsolve, schursolve
from .lssolve import lssolve
from .expintegrator import expintegrator, exponentiate
from .svdsolve import svdsolve
from .bieigsolve import bieigsolve
from .geneigsolve import geneigselector, geneigsolve
from . import factorizations
from .factorizations.blocklanczos import Block

__all__ = [n for n in dir() if not n.startswith("_")]
