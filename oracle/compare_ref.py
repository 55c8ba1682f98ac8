"""Plain-loop restatement of the paired score differences of skyrim_b200/scores.py (``paired_difference_stats``): one
series of per-date differences d_0 .. d_{D-1} at a time, in Python floats, with scipy's Student t functions."""
import math

from scipy.special import stdtr, stdtrit


def paired_stats(d):
    """(mean, ci_low, ci_high, p_value, n_eff) of one series of per-date differences (equally spaced dates)"""
    d = [float(v) for v in d]
    D = len(d)
    nan = float("nan")
    mean = 0.0
    for v in d:
        mean += v
    mean /= D
    if any(math.isnan(v) for v in d):
        return (nan,) * 5
    if D < 3:
        return (mean, nan, nan, nan, nan)
    den = 0.0
    for v in d:
        den += (v - mean) * (v - mean)
    num = 0.0
    for t in range(D - 1):
        num += (d[t] - mean) * (d[t + 1] - mean)
    s = math.sqrt(den / (D - 1))
    r1 = num / den if den > 0.0 else 0.0
    n_eff = D * (1.0 - r1) / (1.0 + r1) if r1 > -1.0 else float(D)
    n_eff = min(max(n_eff, 2.0), float(D))
    if s == 0.0:
        return (mean, mean, mean, 1.0 if mean == 0.0 else 0.0, n_eff)
    se = s / math.sqrt(n_eff)
    p = 2.0 * float(stdtr(n_eff - 1.0, -abs(mean / se)))
    q = float(stdtrit(n_eff - 1.0, 0.975))
    return (mean, mean - q * se, mean + q * se, p, n_eff)
