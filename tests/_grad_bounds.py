"""Per-Gaussian, per-component comparison of the blend backward against the fp64 oracle with rounding-derived bounds
(test infrastructure).

The oracle's blend backward (gof_oracle.render_backward(..., bounds=True)) returns, next to its gradients, two [P,17] error
scales in the order of its accumulator -- dL_dcolors 0-2 | dL_dmean2D 3-5 | dL_dopacity 6 | dL_dv2g 7-16:
  mag       the sum over a Gaussian's pairs of each term's magnitude (every sum and difference taken as the sum of the absolute
            values of its operands), so that a rounding of any intermediate moves the component by a multiple of 2^-24 * mag;
  marginal  the part of mag that depends on a blend decision the host's expf and CUDA's (2 ulp) may take differently.
A blend backward fed with the same forward state passes if, for every Gaussian and component,

    |gpu - oracle|  <=  c * 2^-24 * (1 + L) * mag  +  marginal

with L the longest walk of the view (max n_contrib[0]): T is recovered pair by pair, T * rcp(1 - alpha) on the GPU and
T / (1 - alpha) in the oracle, which drifts by about one ulp per pair.  c is C_BLEND, capped so that c * 2^-24 * (1 + L) never
exceeds 2^-12: a blend backward that needs more than that does not round the way this model says.

C_BLEND is 4x the largest ratio observed on an H100 (1.47, on a 33-Gaussian view whose longest walk is 3 pairs: there the
few roundings inside each pair term outweigh the drift of T), rounded up to a power of two.  Views with walks of hundreds of
pairs stay below 0.08."""
import numpy as np

EPS = 2.0 ** -24
C_BLEND = 8.0


def blend_constant(L):
    """c of the bound for a view whose longest walk is L pairs."""
    return min(C_BLEND, 2.0 ** 12 / (1.0 + float(L)))


def stack17(dcolors, dmeans2D, dopacity, dv2g):
    """The four gradients of the blend backward as one [P,17] float64 array in the oracle's accumulator order."""
    f = lambda a, n: np.asarray(a, np.float64).reshape(-1, n)   # noqa: E731
    return np.concatenate([f(dcolors, 3), f(dmeans2D, 3), f(dopacity, 1), f(dv2g, 10)], axis=1)


def oracle17(d):
    return stack17(d["dL_dcolors"], d["dL_dmean2D"], d["dL_dopacity"], d["dL_dv2g"])


def blend_ratio(got17, ora17, mag, marginal, L):
    """Per entry: the error left after the marginal allowance, in units of 2^-24 * (1 + L) * mag (0 where nothing is left,
    inf where something is left of an entry whose mag is 0).  The comparison passes with constant c iff max <= c."""
    excess = np.maximum(np.abs(got17 - ora17) - marginal, 0.0)
    scale = EPS * (1.0 + float(L)) * mag
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(excess > 0.0, excess / scale, 0.0)
    return np.where((excess > 0.0) & (scale == 0.0), np.inf, r)


def flagged(got17, ora17, mag, marginal, L, c):
    """Indices of the Gaussians with at least one component outside the bound for constant c."""
    return np.nonzero((blend_ratio(got17, ora17, mag, marginal, L) > c).any(axis=1))[0]
