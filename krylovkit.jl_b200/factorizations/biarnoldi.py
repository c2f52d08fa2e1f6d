"""BiArnoldi factorization — mirror of src/factorizations/biarnoldi.jl: two Arnoldi factorizations, one of A
(apply_normal) and one of A' (apply_adjoint), initialised, expanded and shrunk together."""
from __future__ import annotations

from ..algorithms import Orthogonalizer
from ..vectors import B200Vec
from . import arnoldi as ar


class BiArnoldiIterator:
    """BiArnoldiIterator(f, v₀, w₀, orth) — biarnoldi.jl:21-36.  `normal` and `adjoint` are the operators (device
    operators or callables on B200Vec) of the two sides."""

    def __init__(self, normal, adjoint, v0: B200Vec, w0: B200Vec, orth: Orthogonalizer):
        self.iterVH = ar.ArnoldiIterator(normal, v0, orth)
        self.iterWK = ar.ArnoldiIterator(adjoint, w0, orth)


class BiArnoldiFactorization:
    """biarnoldi.jl:1-19: the pair (VH, WK) of ArnoldiFactorizations."""

    def __init__(self, VH: ar.ArnoldiFactorization, WK: ar.ArnoldiFactorization):
        self.VH, self.WK = VH, WK

    def __len__(self):
        return len(self.VH)

    def basis(self):
        return self.VH.basis(), self.WK.basis()

    def rayleighquotient(self):
        return self.VH.rayleighquotient(), self.WK.rayleighquotient()

    def residual(self):
        return self.VH.residual(), self.WK.residual()

    def normres(self):
        return self.VH.normres(), self.WK.normres()


def initialize(it: BiArnoldiIterator) -> BiArnoldiFactorization:
    """initialize(iter) — biarnoldi.jl:55-59."""
    return BiArnoldiFactorization(ar.initialize(it.iterVH), ar.initialize(it.iterWK))


def expand_(it: BiArnoldiIterator, state: BiArnoldiFactorization) -> BiArnoldiFactorization:
    """expand!(iter, state) — biarnoldi.jl:68-75."""
    state.VH = ar.expand_(it.iterVH, state.VH)
    state.WK = ar.expand_(it.iterWK, state.WK)
    return state


def shrink_(state: BiArnoldiFactorization, k: int) -> BiArnoldiFactorization:
    """shrink!(state, k) — biarnoldi.jl:76-83."""
    state.VH = ar.shrink_(state.VH, k)
    state.WK = ar.shrink_(state.WK, k)
    return state
