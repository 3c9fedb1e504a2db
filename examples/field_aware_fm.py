"""Field-aware factorization machine on a small libffm-format stream (needs an H100).

Writes planted one-hot CTR-style data in libffm's text format (``label field:feature:value ...``), reads it back with
``read_libffm``, trains ``DeviceFieldAwareFM`` on the first part and reports the held-out AUC beside a
``DeviceFactorizationMachine`` with the same k and a linear model trained on the same micro-batches: the planted
labels depend on field-aware pair interactions.  ``--optimizer adagrad`` trains all three with libffm's AdaGrad rule
(``--lr 0.2`` is libffm's default rate under it).

    python examples/field_aware_fm.py [--k 4] [--epochs 3] [--optimizer sgd|adagrad] [--lr 0.1]
"""
import argparse
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--optimizer", choices=("sgd", "adagrad"), default="sgd")
    ap.add_argument("--lr", type=float, default=0.1)
    args = ap.parse_args()
    import fps_b200  # noqa: F401
    from fps_b200.models.fm import DeviceFactorizationMachine, DeviceFieldAwareFM, read_libffm, roc_auc
    from fps_b200.utils.synthetic import planted_ffm

    nf, fields, n_train, n_test = 240, 6, 12000, 4000
    rp, cols, flds, labels = planted_ffm(nf, fields, 4, n_train + n_test, seed=3)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "planted.ffm")
        with open(path, "w") as f:
            for e in range(n_train + n_test):
                s = slice(int(rp[e]), int(rp[e + 1]))
                f.write(f"{int(labels[e])} " + " ".join(f"{a}:{b}:1" for a, b in zip(flds[s].tolist(),
                                                                                    cols[s].tolist())) + "\n")
        rp, flds, cols, vals, labels = read_libffm(path)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cols_d, flds_d, vals_d, labels_d = (torch.from_numpy(a).to(dev) for a in (cols, flds, vals, labels))
    t = n_train
    for name in ("FFM", "FM", "linear"):
        if name == "FFM":
            m = DeviceFieldAwareFM(nf, fields, args.k, learning_rate=args.lr, init_range=(-0.1, 0.1), seed=5,
                                   optimizer=args.optimizer)
        else:
            m = DeviceFactorizationMachine(nf, args.k if name == "FM" else 0, learning_rate=args.lr,
                                           init_range=(-0.1, 0.1), seed=5, optimizer=args.optimizer)
        for _ in range(args.epochs):
            m.stats.zero_()
            for b0 in range(0, t, args.batch):
                b1 = min(b0 + args.batch, t)
                r = torch.from_numpy(rp[b0:b1 + 1] - rp[b0]).to(dev)
                s = slice(int(rp[b0]), int(rp[b1]))
                if name == "FFM":
                    m.step_csr(r, cols_d[s], flds_d[s], vals_d[s], labels_d[b0:b1])
                else:
                    m.step_csr(r, cols_d[s], vals_d[s], labels_d[b0:b1])
        st = m.stats.cpu()
        r = torch.from_numpy(rp[t:] - rp[t]).to(dev)
        s = slice(int(rp[t]), None)
        pred = (m.predict_csr(r, cols_d[s], flds_d[s], vals_d[s]) if name == "FFM" else
                m.predict_csr(r, cols_d[s], vals_d[s])).cpu().numpy()
        m.check()
        print(f"{name:6s} k={args.k if name != 'linear' else 0}: last-epoch log loss "
              f"{st[0].item() / st[1].item():.4f}, held-out AUC {roc_auc(pred, labels[t:]):.4f}")
        m.close()


if __name__ == "__main__":
    main()
