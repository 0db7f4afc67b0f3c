"""CPU restatement of the reference's epsilon threshold -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Follows eval_methods.py:186-236 (`find_epsilon`, "Threshold method proposed by Hundman et al.") statement by statement;
the `more_itertools.consecutive_groups` call at :213 only feeds a commented-out variable and is omitted.
Pinned by tests/test_oracle_golden.py against the reference's own function (imported with matplotlib / more_itertools
stubbed) whenever the reference is staged in baseline/_ref."""
import numpy as np


def find_epsilon(errors, reg_level=1):
    e_s = np.asarray(errors)
    best_epsilon = None
    max_score = -10000000
    mean_e_s = np.mean(e_s)                                                    # :193
    sd_e_s = np.std(e_s)                                                       # :194
    for z in np.arange(2.5, 12, 0.5):                                          # :196
        epsilon = mean_e_s + sd_e_s * z
        pruned_e_s = e_s[e_s < epsilon]
        i_anom = np.argwhere(e_s >= epsilon).reshape(-1,)
        buffer = np.arange(1, 50)                                              # :201
        if len(i_anom):
            i_anom = np.concatenate((i_anom, (i_anom[:, None] + buffer).ravel(), (i_anom[:, None] - buffer).ravel()))
        i_anom = i_anom[(i_anom < len(e_s)) & (i_anom >= 0)]
        i_anom = np.sort(np.unique(i_anom))                                    # :210
        if len(i_anom) > 0:
            with np.errstate(all="ignore"):
                mean_perc_decrease = (mean_e_s - np.mean(pruned_e_s)) / mean_e_s if len(pruned_e_s) else np.nan
                sd_perc_decrease = (sd_e_s - np.std(pruned_e_s)) / sd_e_s if len(pruned_e_s) else np.nan
            denom = 1 if reg_level == 0 else (len(i_anom) if reg_level == 1 else len(i_anom) ** 2)
            score = (mean_perc_decrease + sd_perc_decrease) / denom            # :226
            if score >= max_score and len(i_anom) < (len(e_s) * 0.5):
                max_score = score
                best_epsilon = epsilon
    if best_epsilon is None:
        best_epsilon = np.max(e_s)                                             # :233
    return best_epsilon
