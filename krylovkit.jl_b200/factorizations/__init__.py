"""Krylov factorizations (initialize / expand! / shrink!) — mirror of src/factorizations/."""
from .arnoldi import ArnoldiFactorization, ArnoldiIterator
from .biarnoldi import BiArnoldiFactorization, BiArnoldiIterator
from .gkl import GKLFactorization, GKLIterator
from .lanczos import LanczosFactorization, LanczosIterator

__all__ = ["LanczosIterator", "LanczosFactorization", "ArnoldiIterator", "ArnoldiFactorization",
           "BiArnoldiIterator", "BiArnoldiFactorization", "GKLIterator", "GKLFactorization"]
