"""Jaccard / containment -> evolutionary distance (ANI) estimators.

Host-side post-processing of the GPU's integer counts (SURVEY §8 f4): same estimators, argument
names, result classes and thresholds as sourmash/src/sourmash/distance_utils.py (:17-407;
equations of Hera, Pierce-Ward & Koslicki, doi:10.1101/2022.01.11.475870), evaluated in Python
floats in the reference's operation order so that values agree to the last bit.  The only
numerical libraries involved are the ones the reference calls (scipy ``brentq``, ``norm.ppf``,
``binom``).  ``*_matrix`` variants evaluate the point estimates for a whole N x N comparison at
once (numpy), which is what ``compare --ani`` needs after the pairwise-count kernel.
"""
import math
from dataclasses import dataclass, field

import numpy as np


def check_distance(dist):
    "A distance must lie in [0, 1]."
    if not 0 <= dist <= 1:
        raise ValueError(f"Error: distance value {dist :.4f} is not between 0 and 1!")
    return dist


def check_prob_threshold(val, threshold=1e-3):
    "(value, value exceeds threshold) -- likelihood of sharing no hashes by chance alone."
    return val, bool(threshold is not None and val > threshold)


def check_jaccard_error(val, threshold=1e-4):
    return val, bool(threshold is not None and val > threshold)


@dataclass
class ANIResult:
    "Distance / ANI estimated from k-mer containment."
    dist: float
    p_nothing_in_common: float
    p_threshold: float = 1e-3
    size_is_inaccurate: bool = False
    p_exceeds_threshold: bool = field(init=False)

    def check_dist_and_p_threshold(self):
        self.dist = check_distance(self.dist)
        self.p_nothing_in_common, self.p_exceeds_threshold = check_prob_threshold(self.p_nothing_in_common,
                                                                                  self.p_threshold)

    def __post_init__(self):
        self.check_dist_and_p_threshold()

    @property
    def ani(self):
        return None if self.size_is_inaccurate else 1 - self.dist


@dataclass
class jaccardANIResult(ANIResult):
    "ANI from Jaccard; carries the lower bound of the approximation error."
    jaccard_error: float = None
    je_threshold: float = 1e-4

    def __post_init__(self):
        self.check_dist_and_p_threshold()
        if self.jaccard_error is None:
            raise ValueError("Error: jaccard_error cannot be None.")
        self.jaccard_error, self.je_exceeds_threshold = check_jaccard_error(self.jaccard_error, self.je_threshold)

    @property
    def ani(self):
        if self.je_exceeds_threshold or self.size_is_inaccurate:   # estimate not trustworthy
            return None
        return 1 - self.dist


@dataclass
class ciANIResult(ANIResult):
    "ANI from containment with an optional confidence interval."
    dist_low: float = None
    dist_high: float = None

    def __post_init__(self):
        self.check_dist_and_p_threshold()
        if self.dist_low is not None and self.dist_high is not None:
            self.dist_low = check_distance(self.dist_low)
            self.dist_high = check_distance(self.dist_high)

    @property
    def ani_low(self):
        if self.dist_high is None or self.size_is_inaccurate:
            return None
        return 1 - self.dist_high

    @property
    def ani_high(self):
        if self.dist_low is None or self.size_is_inaccurate:
            return None
        return 1 - self.dist_low


# ------------------------------------------------------------------------------ mutation model
def r1_to_q(k, r1):
    "Probability that a k-mer carries at least one mutation at per-base rate r1."
    r1 = float(r1)
    return float(1 - (1 - r1) ** k)


def var_n_mutated(L, k, r1, *, q=None):
    "Variance of the number of mutated k-mers among L."
    if r1 == 0:
        return 0.0
    r1 = float(r1)
    if q is None:
        q = r1_to_q(k, r1)
    varN = (L * (1 - q) * (q * (2 * k + (2 / r1) - 1) - 2 * k)
            + k * (k - 1) * (1 - q) ** 2
            + (2 * (1 - q) / (r1 ** 2)) * ((1 + (k - 1) * (1 - q)) * r1 - q))
    if varN < 0.0:
        raise ValueError("Error: varN <0.0!")
    return float(varN)


def exp_n_mutated(L, k, r1):
    return L * r1_to_q(k, r1)


def exp_n_mutated_squared(L, k, p):
    return var_n_mutated(L, k, p) + exp_n_mutated(L, k, p) ** 2


def probit(p):
    from scipy.stats import norm
    return norm.ppf(p)


def handle_seqlen_nkmers(ksize, *, sequence_len_bp=None, n_unique_kmers=None):
    if n_unique_kmers is not None:
        return n_unique_kmers
    if sequence_len_bp is None:
        raise ValueError("Error: distance estimation requires input of either 'sequence_len_bp' or 'n_unique_kmers'")
    return sequence_len_bp - (ksize - 1)


def set_size_chernoff(set_size, scaled, *, relative_error=0.05):
    "Two-sided Chernoff bound on |sketch_size * scaled - set_size| <= relative_error * set_size."
    return 1 - 2 * np.exp(-(relative_error ** 2) * set_size / (scaled * 3))


def set_size_exact_prob(set_size, scaled, *, relative_error=0.05):
    """Exact probability that sketch_size * scaled is within relative_error of set_size
    (sketch_size ~ Binomial(set_size, 1/scaled))."""
    from scipy.stats import binom
    lo = -set_size / scaled * (relative_error - 1)
    hi = set_size / scaled * (relative_error + 1)
    if lo == int(lo):             # an integral lower edge belongs to the interval
        return (binom.cdf(hi, set_size, 1 / scaled) - binom.cdf(lo, set_size, 1 / scaled)
                + binom.pmf(lo, set_size, 1 / scaled))
    return binom.cdf(hi, set_size, 1 / scaled) - binom.cdf(lo, set_size, 1 / scaled)


def get_expected_log_probability(n_unique_kmers, ksize, mutation_rate, scaled_fraction):
    "log P(no unmutated k-mer is sampled); scaled_fraction = 1/scaled."
    exp_nmut = exp_n_mutated(n_unique_kmers, ksize, mutation_rate)
    try:
        return (n_unique_kmers - exp_nmut) * math.log(1.0 - scaled_fraction)
    except Exception:
        return float("-inf")


def get_exp_probability_nothing_common(mutation_rate, ksize, scaled, *, n_unique_kmers=None, sequence_len_bp=None):
    "Expected probability that a sketch and the sketch of its mutated copy share nothing."
    n_unique_kmers = handle_seqlen_nkmers(ksize, sequence_len_bp=sequence_len_bp, n_unique_kmers=n_unique_kmers)
    f_scaled = 1.0 / float(scaled)
    if mutation_rate == 1.0:
        return 1.0
    if mutation_rate == 0.0:
        return 0.0
    return math.exp(get_expected_log_probability(n_unique_kmers, ksize, mutation_rate, f_scaled))


# ------------------------------------------------------------------------------ estimators
def containment_to_distance(containment, ksize, scaled, *, n_unique_kmers=None, sequence_len_bp=None,
                            confidence=0.95, estimate_ci=False, prob_threshold=1e-3):
    "Containment -> distance (point estimate, optional confidence interval)."
    sol1 = sol2 = point_estimate = None
    n_unique_kmers = handle_seqlen_nkmers(ksize, sequence_len_bp=sequence_len_bp, n_unique_kmers=n_unique_kmers)
    if containment == 0:
        point_estimate = sol1 = sol2 = 1.0
    elif containment == 1:
        point_estimate = sol1 = sol2 = 0.0
    else:
        point_estimate = 1.0 - containment ** (1.0 / ksize)
        if estimate_ci:
            try:
                from scipy.optimize import brentq
                alpha = 1 - confidence
                z_alpha = probit(1 - alpha / 2)
                f_scaled = 1.0 / scaled
                bias_factor = 1 - (1 - f_scaled) ** n_unique_kmers
                term_1 = (1.0 - f_scaled) / (f_scaled * n_unique_kmers ** 3 * bias_factor ** 2)

                def var_direct(pest):
                    term_2 = (n_unique_kmers * exp_n_mutated(n_unique_kmers, ksize, pest)
                              - exp_n_mutated_squared(n_unique_kmers, ksize, pest))
                    term_3 = var_n_mutated(n_unique_kmers, ksize, pest) / n_unique_kmers ** 2
                    return term_1 * term_2 + term_3

                def upper(pest):
                    return (1 - pest) ** ksize + z_alpha * np.sqrt(var_direct(pest)) - containment

                def lower(pest):
                    return (1 - pest) ** ksize - z_alpha * np.sqrt(var_direct(pest)) - containment

                sol1 = brentq(upper, 0.0000001, 0.9999999)
                sol2 = brentq(lower, 0.0000001, 0.9999999)
            except ValueError:
                # happens with very small sketches only: no interval
                sol1 = sol2 = None
    prob_nothing_in_common = get_exp_probability_nothing_common(point_estimate, ksize, scaled,
                                                                n_unique_kmers=n_unique_kmers)
    return ciANIResult(point_estimate, prob_nothing_in_common, dist_low=sol2, dist_high=sol1,
                       p_threshold=prob_threshold)


def jaccard_to_distance(jaccard, ksize, scaled, *, n_unique_kmers=None, sequence_len_bp=None,
                        prob_threshold=1e-3, err_threshold=1e-4):
    "Jaccard -> distance point estimate plus a lower bound of the approximation error."
    n_unique_kmers = handle_seqlen_nkmers(ksize, sequence_len_bp=sequence_len_bp, n_unique_kmers=n_unique_kmers)
    if jaccard == 0:
        point_estimate, error_lower_bound = 1.0, 0.0
    elif jaccard == 1:
        point_estimate, error_lower_bound = 0.0, 0.0
    else:
        point_estimate = 1.0 - (2.0 * jaccard / float(1 + jaccard)) ** (1.0 / float(ksize))
        exp_n_mut = exp_n_mutated(n_unique_kmers, ksize, point_estimate)
        var_n_mut = var_n_mutated(n_unique_kmers, ksize, point_estimate)
        error_lower_bound = 1.0 * n_unique_kmers * var_n_mut / (n_unique_kmers + exp_n_mut) ** 3
    prob_nothing_in_common = get_exp_probability_nothing_common(point_estimate, ksize, scaled,
                                                                n_unique_kmers=n_unique_kmers)
    return jaccardANIResult(point_estimate, prob_nothing_in_common, jaccard_error=error_lower_bound,
                            p_threshold=prob_threshold, je_threshold=err_threshold)


# ------------------------------------------------------------------------------ whole matrices
def _pow(values, exponent):
    """values ** exponent, element by element with the C library's pow -- bit-identical to the Python floats of the
    per-pair formulas (numpy's vectorised power is allowed to differ in the last bit)."""
    from ._lowlevel import ffi, lib
    a = np.ascontiguousarray(values, dtype=np.float64)
    out = np.empty_like(a)
    lib.smb_pow_f64(ffi.cast("double *", a.ctypes.data), float(exponent), ffi.cast("double *", out.ctypes.data), a.size)
    return out


def jaccard_to_ani_matrix(jaccard, sizes, ksize, scaled, *, err_threshold=1e-4, prob_threshold=1e-3,
                          size_accurate=None, cells=None):
    """ANI for every pair of an N x N Jaccard matrix (what ``compare --ani`` reports:
    compare.py:36-54 -> MinHash.jaccard_ani).  ``sizes[i]`` = number of hashes of sketch i.
    Untrustworthy estimates (error bound above err_threshold, or a sketch whose size estimate
    is inaccurate) become 0.0 like in compare_serial; the diagonal is 1.0.  ``cells`` (bool N x N) limits the two warning
    flags to those pairs (a caller that keeps only part of the matrix).
    Returns (ani, jaccard_ani_untrustworthy, potential_false_negatives)."""
    J = np.asarray(jaccard, dtype=np.float64)
    n = J.shape[0]
    sizes = np.asarray(sizes, dtype=np.float64)
    L = np.rint((sizes[:, None] + sizes[None, :]) / 2 * scaled)          # round(avg sketch size * scaled)
    k = float(ksize)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = 1.0 - _pow(2.0 * J / (1 + J), 1.0 / k)
        r = np.where(J == 0, 1.0, np.where(J == 1, 0.0, r))
        q = 1 - _pow(1 - r, ksize)
        var = (L * (1 - q) * (q * (2 * k + (2 / r) - 1) - 2 * k) + k * (k - 1) * (1 - q) ** 2
               + (2 * (1 - q) / (r ** 2)) * ((1 + (k - 1) * (1 - q)) * r - q))
        var = np.where(r == 0, 0.0, var)
        err = np.where((J == 0) | (J == 1), 0.0, 1.0 * L * var / (L + L * q) ** 3)
        p_nothing = np.exp((L - L * q) * math.log(1.0 - 1.0 / float(scaled)))
        p_nothing = np.where(r == 1.0, 1.0, np.where(r == 0.0, 0.0, p_nothing))
    bad = err > err_threshold
    if size_accurate is not None:
        acc = np.asarray(size_accurate, dtype=bool)
        bad = bad | ~(acc[:, None] & acc[None, :])
    ani = np.where(bad, 0.0, 1.0 - r)
    off = ~np.eye(n, dtype=bool)
    if cells is not None:
        off &= np.asarray(cells, dtype=bool)
    untrustworthy = bool((err > err_threshold)[off].any())
    false_neg = bool((p_nothing > prob_threshold)[off].any())
    np.fill_diagonal(ani, 1.0)
    return ani, untrustworthy, false_neg


def containment_to_ani_matrix(containment, ksize, *, size_accurate_rows=None, size_accurate_cols=None):
    "Point-estimate ANI 1 - (1 - c**(1/k)) for a matrix of containments (no intervals)."
    C = np.asarray(containment, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = 1.0 - _pow(C, 1.0 / ksize)
    r = np.where(C == 0, 1.0, np.where(C == 1, 0.0, r))
    ani = 1.0 - r
    if size_accurate_rows is not None and size_accurate_cols is not None:
        ok = np.asarray(size_accurate_rows, bool)[:, None] & np.asarray(size_accurate_cols, bool)[None, :]
        ani = np.where(ok, ani, 0.0)
    return ani
