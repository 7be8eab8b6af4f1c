"""The selection rule of multi-hypothesis alignment (dvo_b200_match_batch_hypotheses, include/dvo_b200.h), restated in Python
from its definition: the score of a screened hypothesis from the level statistics of its screening level, and the choice."""
import math


def score(level, min_ratio):
    """per-constraint negative log-likelihood of one hypothesis, or NaN if it is not eligible.  level: the dvo_b200_level_stats
    of the screening level as a dict (Result.levels[i])"""
    if not level["has_iteration_with_increment"]:
        return math.nan
    n = level["last_increment_valid_constraints"]
    try:
        ratio = float(n) / float(level["valid_pixels"])
    except ZeroDivisionError:
        ratio = math.nan if n == 0 else math.copysign(math.inf, n)
    if not ratio >= min_ratio:
        return math.nan
    try:
        s = level["last_increment_log_likelihood"] / float(n)
    except ZeroDivisionError:
        return math.nan   # 0 constraints: x / 0 is never finite
    return s if math.isfinite(s) else math.nan


def pick(scores):
    """the eligible hypothesis with the smallest score, the lowest index on a tie; 0 if none is eligible"""
    best = None
    for j, s in enumerate(scores):
        if not math.isnan(s) and (best is None or s < scores[best]):
            best = j
    return 0 if best is None else best
