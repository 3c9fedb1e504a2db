"""Factorization machine on planted one-hot CTR-style data (needs an H100).

Trains ``DeviceFactorizationMachine`` with k factors and the same model with ``num_factors=0`` (plain logistic
regression) on the same micro-batches, then reports the held-out AUC of both: the planted labels depend on
pairwise feature interactions, which only the factors can model.

    python examples/factorization_machine.py [--k 4] [--epochs 3]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    import fps_b200  # noqa: F401
    from fps_b200.models.fm import DeviceFactorizationMachine, roc_auc
    from fps_b200.utils.synthetic import planted_fm

    nf, fields, n_train, n_test = 240, 6, 12000, 4000
    rp, cols, labels = planted_fm(nf, fields, 4, n_train + n_test, seed=3, loss="logistic")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cols_d, labels_d = cols.to(dev), labels.to(dev)
    for k in (args.k, 0):
        m = DeviceFactorizationMachine(nf, k, loss="logistic", learning_rate=0.05, init_range=(-0.1, 0.1), seed=5)
        for _ in range(args.epochs):
            m.stats.zero_()
            for b0 in range(0, n_train, args.batch):
                b1 = min(b0 + args.batch, n_train)
                m.step_csr((rp[b0:b1 + 1] - rp[b0]).to(dev), cols_d[rp[b0]:rp[b1]], None, labels_d[b0:b1])
        s = m.stats.cpu()
        pred = m.predict_csr((rp[n_train:] - rp[n_train]).to(dev), cols_d[rp[n_train]:]).cpu()
        m.check()
        print(f"k={k}: last-epoch log loss {s[0].item() / s[1].item():.4f}, held-out AUC "
              f"{roc_auc(pred.numpy(), labels[n_train:].numpy()):.4f}")
        m.close()


if __name__ == "__main__":
    main()
