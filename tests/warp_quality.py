"""The WARP quality gate (tests/test_mf_warp_host.py, tests/test_gpu_mf_warp.py, tests/mp_warp_check.py): the
``lowrank_implicit`` set, metrics, epochs and L2 weight of tests/bpr_quality.py, up to ``T`` candidates per positive,
the margin and the rate below.

WARP scales each step by ``L = ln((N - 1) // n)``, up to ln(599) = 6.4 here, so it takes a smaller rate than BPR.
Sequential numpy runs, 30 epochs, held-out AUC / recall@10 (random: 0.5 / ~0.017):

    WARP lr 0.01: 0.743 / 0.097      BPR lr 0.01: 0.517 / 0.025
    WARP lr 0.1:  0.521 / 0.025      BPR lr 0.1:  0.743 / 0.110
    (WARP at lr 0.1 diverges: max |u| reaches 5e28)
"""
import numpy as np
import torch

from tests import bpr_quality as Q

T, MARGIN, LR = 10, 1.0, 0.01
AUC_GATE, RECALL_GATE = 0.68, 0.07


def train_numpy(tu, ti, lr=LR):
    """Sequential WARP with :func:`warp_delta`, candidates uniform over the items (the positive is void)."""
    from fps_b200.models.mf.common import warp_delta

    rng = np.random.default_rng(0)
    U = rng.uniform(-Q.INIT, Q.INIT, (Q.NUM_USERS, Q.K)); V = rng.uniform(-Q.INIT, Q.INIT, (Q.NUM_ITEMS, Q.K))
    tu, ti = tu.numpy(), ti.numpy()
    for _ in range(Q.EPOCHS):
        for u, i, cand in zip(tu, ti, rng.integers(0, Q.NUM_ITEMS, (tu.size, T))):
            rows = [None if j == i else V[j] for j in cand]
            du, dvi, t, dvj, _, _, _ = warp_delta(U[u], V[i], rows, MARGIN, lr, Q.REG, Q.NUM_ITEMS)
            if t is None:
                continue
            U[u] += du; V[i] += dvi; V[cand[t]] += dvj
    return torch.from_numpy(U), torch.from_numpy(V)
