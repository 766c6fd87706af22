"""The reference fixture of the training inputs' synthetic errors (tests/golden/inputs.npz) and the two-sample
chi-square comparison both the oracle's and the device's samples are held to."""
import os

import numpy as np
from scipy.stats import chi2_contingency

from oracle import inputs_oracle as io

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "inputs.npz"))
CASES = [str(n) for n in GOLDEN["case_names"]]
CLOSE = "close_pairs"          # sources overlap: compared on the 2-D offset grid as well
SEEDS = (0x5EED_0001_2345_6789, 0x0000_00AB_CDEF_0123)
P_FAIL = 1e-4


def case(name):
    i = CASES.index(name)
    return GOLDEN["case_joints"][i], float(GOLDEN["case_area"][i]), i


def chi2_p(ref, got):
    """p-value of the homogeneity of two count vectors; cells with expected count < 5 are pooled into one."""
    tab = np.stack([ref, got]).astype(np.float64)
    tab = tab[:, tab.sum(0) > 0]
    small = tab.sum(0) * 0.5 < 5
    if small.any():
        pooled = tab[:, small].sum(1, keepdims=True)
        tab = np.concatenate([tab[:, ~small], pooled], 1)
        if pooled.sum() * 0.5 < 5 and tab.shape[1] > 2:   # still small: merge it into the last regular cell
            tab = np.concatenate([tab[:, :-2], tab[:, -2:].sum(1, keepdims=True)], 1)
    if tab.shape[1] < 2:
        return 1.0
    return float(chi2_contingency(tab)[1])


def fixture_pvalues(name, out):
    """Per-joint p-values of samples out [M, 17, 3] of case `name` against the reference's counts: the annulus cells,
    and for the close-pair case the offset grid too.  -> list of (p, label)."""
    joints, area, i = case(name)
    ps = []
    got = io.histogram(io.outcome_cells(out, joints, area), io.N_CELL)
    for j in range(17):
        ps.append((chi2_p(GOLDEN["ref_cells"][i, j], got[j]), f"{name} joint {j} annuli"))
    if name == CLOSE:
        got2 = io.histogram(io.offset_cells(out, joints, area), io.N_CELL_2D)
        for j in range(17):
            ps.append((chi2_p(GOLDEN["ref_offsets"][i, j], got2[j]), f"{name} joint {j} offsets"))
    return ps


def error_table():
    """The reference's noise_stats table as its list of dicts, and Human36M's joint order."""
    table = [{"Joint": str(n), "mean": tuple(m), "std": tuple(s), "weight": float(w)}
             for n, m, s, w in zip(GOLDEN["error_joint"], GOLDEN["error_mean"], GOLDEN["error_std"],
                                   GOLDEN["error_weight"])]
    return table, [str(n) for n in GOLDEN["h36m_joints_name"]]


def ordered_table():
    """(mean [17, 2], std [17, 2], weight [17]) in Human36M's joint order (get_stat)."""
    table, names = error_table()
    rows = [next(e for e in table if e["Joint"] == n) for n in names]
    return (np.array([r["mean"] for r in rows]), np.array([r["std"] for r in rows]),
            np.array([r["weight"] for r in rows]))
