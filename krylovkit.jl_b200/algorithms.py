"""Algorithm parameter structs and Orthogonalizer tags — mirror of src/algorithms.jl.

Only the contract is mirrored (names, defaults, meaning); the tags select the kernel
variant in libb200krylov (B2K_CGS ... B2K_MGSIR).
"""
from __future__ import annotations

from dataclasses import dataclass, field

from . import _lib as L

# verbosity levels — src/KrylovKit.jl:159-162
SILENT_LEVEL, WARN_LEVEL, STARTSTOP_LEVEL, EACHITERATION_LEVEL = 0, 1, 2, 3


# ---- Orthogonalizer hierarchy — src/algorithms.jl:17-80 -----------------------------
@dataclass(frozen=True)
class Orthogonalizer:
    tag: int = -1
    eta: float = 0.0

    @property
    def is_reorth2(self) -> bool:      # Union{ClassicalGramSchmidt2, ModifiedGramSchmidt2}
        return self.tag in (L.CGS2, L.MGS2, L.MGS2B)

    @property
    def is_ir(self) -> bool:           # Union{ClassicalGramSchmidtIR, ModifiedGramSchmidtIR}
        return self.tag in (L.CGSIR, L.MGSIR)


@dataclass(frozen=True)
class ClassicalGramSchmidt(Orthogonalizer):
    tag: int = L.CGS


@dataclass(frozen=True)
class ModifiedGramSchmidt(Orthogonalizer):
    tag: int = L.MGS


@dataclass(frozen=True)
class ClassicalGramSchmidt2(Orthogonalizer):
    tag: int = L.CGS2


@dataclass(frozen=True)
class ModifiedGramSchmidt2(Orthogonalizer):
    tag: int = L.MGS2


@dataclass(frozen=True)
class ModifiedGramSchmidt2Blocked(Orthogonalizer):
    """Engine-specific, FLAGGED — not a KrylovKit orthogonalizer.  ModifiedGramSchmidt2 with every sweep over the
    whole basis applied as ONE classical block (include/b200krylov.h B2K_MGS2B): the reference default's two
    orthogonalisations at the speed of ClassicalGramSchmidt2.  In the Lanczos recurrence the two-vector first part
    (β v₋ removed, then α = ⟨v, w⟩, lanczos.jl:326-328) is exactly the reference's; the second sweep over all of V
    takes its coefficients from one vector instead of k successively updated ones — a rounding-level change."""
    tag: int = L.MGS2B


@dataclass(frozen=True)
class ClassicalGramSchmidtIR(Orthogonalizer):
    tag: int = L.CGSIR
    eta: float = 1.0 / 2.0 ** 0.5       # algorithms.jl:67


@dataclass(frozen=True)
class ModifiedGramSchmidtIR(Orthogonalizer):
    tag: int = L.MGSIR
    eta: float = 1.0 / 2.0 ** 0.5       # algorithms.jl:80


cgs, mgs, cgs2, mgs2 = (ClassicalGramSchmidt(), ModifiedGramSchmidt(), ClassicalGramSchmidt2(),
                        ModifiedGramSchmidt2())
cgsr, mgsr = ClassicalGramSchmidtIR(), ModifiedGramSchmidtIR()
mgs2b = ModifiedGramSchmidt2Blocked()          # flagged engine mode, see the class


# ---- KrylovDefaults — src/algorithms.jl:556-564 -------------------------------------
class KrylovDefaults:
    orth: Orthogonalizer = mgs2
    krylovdim: int = 30
    maxiter: int = 100
    tol: float = 1e-12
    verbosity: int = WARN_LEVEL


# ---- algorithm structs — src/algorithms.jl:110-521 (the ones on the scoped path) ----
@dataclass(frozen=True)
class Lanczos:
    orth: Orthogonalizer = field(default_factory=lambda: KrylovDefaults.orth)
    krylovdim: int = KrylovDefaults.krylovdim
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    eager: bool = False
    verbosity: int = KrylovDefaults.verbosity


@dataclass(frozen=True)
class BlockLanczos:
    """src/algorithms.jl:152-171.  krylovdim defaults to KrylovDefaults.blockkrylovdim = 100;
    `qr_tol` is the rank tolerance of block_qr!."""
    orth: Orthogonalizer = field(default_factory=lambda: KrylovDefaults.orth)
    krylovdim: int = 100
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    qr_tol: float = KrylovDefaults.tol
    eager: bool = False
    verbosity: int = KrylovDefaults.verbosity
    # Engine-specific, FLAGGED (default: the reference's arithmetic): block-classical Gram-Schmidt twice + CholeskyQR2
    # instead of the modified Gram-Schmidt loops of block_reorthogonalize! / block_qr! — factorizations/blocklanczos.py
    fast_block: bool = False


@dataclass(frozen=True)
class Arnoldi:
    orth: Orthogonalizer = field(default_factory=lambda: KrylovDefaults.orth)
    krylovdim: int = KrylovDefaults.krylovdim
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    eager: bool = False
    verbosity: int = KrylovDefaults.verbosity


@dataclass(frozen=True)
class BiArnoldi:
    """src/algorithms.jl:255-291: the two-sided Krylov-Schur method of bieigsolve."""
    orth: Orthogonalizer = field(default_factory=lambda: KrylovDefaults.orth)
    krylovdim: int = KrylovDefaults.krylovdim
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    eager: bool = False
    verbosity: int = KrylovDefaults.verbosity


@dataclass(frozen=True)
class GKL:
    orth: Orthogonalizer = field(default_factory=lambda: KrylovDefaults.orth)
    krylovdim: int = KrylovDefaults.krylovdim
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    eager: bool = False
    verbosity: int = KrylovDefaults.verbosity
    # flagged, not a reference field: one pass over a dense device operator per GKL step instead of two
    # (factorizations/gkl.py); coefficients differ from the reference step by rounding only
    onepass: bool = False


@dataclass(frozen=True)
class GMRES:
    orth: Orthogonalizer = field(default_factory=lambda: KrylovDefaults.orth)
    maxiter: int = KrylovDefaults.maxiter
    krylovdim: int = KrylovDefaults.krylovdim
    tol: float = KrylovDefaults.tol
    verbosity: int = KrylovDefaults.verbosity


@dataclass(frozen=True)
class CG:
    """src/algorithms.jl:344-355."""
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    verbosity: int = KrylovDefaults.verbosity


@dataclass(frozen=True)
class BiCGStab:
    """src/algorithms.jl:457-481."""
    maxiter: int = KrylovDefaults.maxiter
    tol: float = KrylovDefaults.tol
    verbosity: int = KrylovDefaults.verbosity


@dataclass(frozen=True)
class LSMR:
    """src/algorithms.jl:483-521.  `krylovdim` = how many recent right vectors the next one is
    reorthogonalised against; the default orthogonalizer is plain MGS (:517)."""
    orth: Orthogonalizer = mgs
    maxiter: int = KrylovDefaults.maxiter
    krylovdim: int = KrylovDefaults.krylovdim
    tol: float = KrylovDefaults.tol
    verbosity: int = KrylovDefaults.verbosity


@dataclass
class ConvergenceInfo:
    """src/KrylovKit.jl:212-218.  numops = operator applications, numiter = restart cycles."""
    converged: int
    residual: object
    normres: object
    numiter: int
    numops: int
