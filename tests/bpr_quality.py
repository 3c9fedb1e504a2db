"""Shared data and metrics of the BPR quality gates (tests/test_mf_bpr_host.py, tests/test_gpu_mf_bpr.py,
tests/mp_bpr_check.py): a small ``lowrank_implicit`` set, held-out sampled AUC and recall@10 with each
user's train items excluded, and the gate a sequential numpy BPR run clears with margin."""
import numpy as np
import torch

NUM_USERS, NUM_ITEMS, PER_USER, HELD_OUT, SEED = 400, 600, 20, 5, 3
K, LR, REG, EPOCHS, INIT = 16, 0.1, 0.01, 30, 0.1
# The sequential numpy run below reaches AUC 0.744 and recall@10 0.110 (random: 0.5 and ~0.017).
AUC_GATE, RECALL_GATE = 0.68, 0.07


def data():
    from fps_b200.utils.synthetic import lowrank_implicit

    return lowrank_implicit(NUM_USERS, NUM_ITEMS, PER_USER, HELD_OUT, SEED)


def metrics(U: torch.Tensor, V: torch.Tensor, train, test, n_neg: int = 50, seed: int = 1):
    """``(auc, recall@10)`` of the factor matrices ``U`` [users, k] / ``V`` [items, k] (any device):
    AUC over each held-out pair against ``n_neg`` random items the user has not consumed, recall@10 of
    the top-10 list without the user's train items."""
    U, V = U.double().cpu(), V.double().cpu()
    (tu, ti), (eu, ei) = train, test
    nu, ni = U.shape[0], V.shape[0]
    S = U @ V.T
    tm = torch.zeros(nu, ni, dtype=torch.bool); tm[tu, ti] = True
    em = torch.zeros(nu, ni, dtype=torch.bool); em[eu, ei] = True
    jn = torch.randint(0, ni, (eu.numel(), n_neg), generator=torch.Generator().manual_seed(seed))
    valid = ~(tm[eu[:, None], jn] | em[eu[:, None], jn])
    auc = (((S[eu, ei][:, None] > S[eu[:, None], jn]) & valid).sum() / valid.sum()).item()
    top = S.masked_fill(tm, -float("inf")).topk(10, 1).indices
    return auc, em.gather(1, top).sum().item() / eu.numel()


def train_numpy(tu, ti):
    """Sequential BPR with :func:`bpr_delta`, one uniform negative (never the positive) per positive."""
    from fps_b200.models.mf.common import bpr_delta

    rng = np.random.default_rng(0)
    U = rng.uniform(-INIT, INIT, (NUM_USERS, K)); V = rng.uniform(-INIT, INIT, (NUM_ITEMS, K))
    tu, ti = tu.numpy(), ti.numpy()
    for _ in range(EPOCHS):
        for u, i, j in zip(tu, ti, rng.integers(0, NUM_ITEMS, tu.size)):
            if j == i:
                continue
            du, dvi, dvj, _ = bpr_delta(U[u], V[i], V[j], LR, REG)
            U[u] += du; V[i] += dvi; V[j] += dvj
    return torch.from_numpy(U), torch.from_numpy(V)
