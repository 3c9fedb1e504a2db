#!/usr/bin/env python
"""CBOW from a token stream: the fused CBOW kernel (``DeviceSkipGram.train_tokens(cbow=True)``) against the fused
skip-gram kernel on the same corpus, and against a CBOW written in stock PyTorch on the same compaction, radii and
noise words, on one GPU.

    python benchmarks/w2v_cbow_bench.py [--out profiles/h100_w2v_cbow_bench.json]

Shape: that of ``w2v_tokens_bench.py``: 1M words x 300, ``negative=5`` (unigram noise from the corpus counts),
``window=5``, ``sample=1e-3``, a Zipf ``topic_corpus`` of about 3.1M tokens per call.  Records, in one process:

* the card (name, power limit, max SM clock), before and after;
* per path, ms per call, words per second and target updates per second: fused CBOW (its two kernels), fused
  skip-gram, and the torch CBOW (gather, segment mean with ``index_add_``, batched dots, ``index_add_`` pushes, in
  chunks of centers), and the CBOW kernel alone;
* TB/s by the bytes model (DESIGN §2.14): a CBOW center moves each of its ``cw`` context rows twice and each target
  row twice; a skip-gram center moves its own row twice and each target row twice.

The paths are alternated round by round; the median and the spread over the rounds are kept.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "benchmarks"))

from w2v_tokens_bench import _events, _philox_np, _summary, card  # noqa: E402

VOCAB, DIM, NEG, WINDOW, SAMPLE = 1_000_000, 300, 5, 5, 1e-3
TOPICS, SENT_LEN, SENTENCES = 1000, 20, 150_000
LR = 0.025
CHUNK = 1 << 18   # centers per torch chunk


def noise_words(pos, centers, cdf, last, step, seed):
    """The kernel's noise words of each center (context slot 0): tries 0 and 1 of word j from counter
    ``(i, 2, j, step)``, through the fp64 CDF, rejected against the center; -1 when both hit it (the kernel would
    try further, which at this vocabulary happens for no center here; the count is recorded)."""
    out = np.empty((len(pos), NEG), dtype=np.int64)
    total = float(cdf[-1])
    for j in range(NEG):
        x, y, z, w = _philox_np(pos, 2, j, step, seed & 0xFFFFFFFF, seed >> 32)
        picks = []
        for hi, lo in ((x, y), (z, w)):
            h = (hi.astype(np.uint64) << np.uint64(32)) | lo.astype(np.uint64)
            u = (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 * total
            c = np.searchsorted(cdf, u, side="right")
            picks.append(np.where(c < len(cdf), c, last))
        out[:, j] = np.where(picks[0] != centers, picks[0], np.where(picks[1] != centers, picks[1], -1))
    return out


def context_index(seq, n, radius):
    """Per live center (a kept word with at least one context): its entry and, flattened, (center slot, context
    entry) pairs in increasing position."""
    s = seq[:n].long()
    seg = torch.cumsum((s < 0).long(), 0)
    idx = torch.arange(n, device=s.device)
    oks, qs = [], []
    for o in list(range(-WINDOW, 0)) + list(range(1, WINDOW + 1)):
        q = (idx + o).clamp(0, n - 1)
        ok = (s >= 0) & (idx + o >= 0) & (idx + o < n) & (s[q] >= 0) & (seg[q] == seg) & (radius >= abs(o))
        oks.append(ok); qs.append(q)
    ok, q = torch.stack(oks, 1), torch.stack(qs, 1)          # [n, 2W]
    cw = ok.sum(1)
    live = torch.nonzero(cw > 0).flatten()
    return live, ok[live], q[live], cw[live]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_w2v_cbow_bench.json"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    import fps_b200  # noqa: F401
    from fps_b200.models.w2v import DeviceSkipGram
    from fps_b200.models.w2v_ref import radii
    from fps_b200.ops import native
    from fps_b200.utils.synthetic import topic_corpus

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"card_before": card(), "shape": dict(vocab=VOCAB, dim=DIM, negative=NEG, window=WINDOW, sample=SAMPLE,
                                                 topics=TOPICS, sentence_len=SENT_LEN, sentences=SENTENCES, lr=LR)}
    tok_h = topic_corpus(VOCAB, TOPICS, SENT_LEN, SENTENCES, seed=1)
    counts = np.bincount(tok_h[tok_h >= 0].numpy(), minlength=VOCAB).astype(np.float64)
    tok = tok_h.to(dev)
    n_tok = tok.numel()
    m = DeviceSkipGram(VOCAB, DIM, learning_rate=LR, negative=NEG, seed=1, word_counts=counts,
                       noise_counts=counts, sample=SAMPLE)
    step0 = m.step_no
    # the torch CBOW trains the centers of the fused path's first call: same compaction, radii and noise words
    seq, pos, n_comp = native.w2v_subsample(tok, VOCAB, m._keep_p, seed=m.seed, step=step0)
    n = int(n_comp.item())
    pos_h = pos[:n].cpu().numpy()
    rad = torch.from_numpy(radii(pos_h, WINDOW, step0, m.seed, _philox_np)).to(dev)
    live, ok, q, cw = context_index(seq, n, rad)
    centers = seq[:n].long()[live]
    noise = noise_words(pos_h[live.cpu().numpy()].astype(np.int64), centers.cpu().numpy(),
                        m._noise_cdf.cpu().numpy(), m._noise_last, step0, m.seed)
    voids = int((noise < 0).sum())
    targets = torch.cat([centers[:, None], torch.from_numpy(noise).to(dev)], 1)          # [live, 1 + NEG]
    labels = torch.zeros(1, 1 + NEG, device=dev)
    labels[0, 0] = 1.0
    ctx_words = seq[:n].long()[q]                                                         # [live, 2W]
    n_live, n_ctx = live.numel(), int(cw.sum())
    W_in = m.w_in.local[:VOCAB, :DIM].clone()
    W_out = m.w_out.local[:VOCAB, :DIM].clone()
    chunks = [(lo, min(lo + CHUNK, n_live)) for lo in range(0, n_live, CHUNK)]

    def torch_cbow():
        for lo, hi in chunks:
            okc, cwc, tg = ok[lo:hi], cw[lo:hi], targets[lo:hi]
            slot, k = torch.nonzero(okc, as_tuple=True)
            words = ctx_words[lo:hi][slot, k]
            h = torch.zeros(hi - lo, DIM, device=dev).index_add_(0, slot, W_in[words]) / cwc[:, None]
            valid = tg >= 0
            V = W_out[tg.clamp_min(0)]                                                    # [c, 1 + NEG, D]
            d = torch.bmm(V, h[:, :, None]).squeeze(2)
            g = LR * (labels - torch.sigmoid(d)) * valid
            e = torch.bmm(g[:, None, :], V).squeeze(1)
            W_out.index_add_(0, tg[valid], (g[:, :, None] * h[:, None, :])[valid])
            W_in.index_add_(0, words, e[slot])

    def fused_cbow():
        m.train_tokens(tok, window=WINDOW, cbow=True)

    def fused_sg():
        m.train_tokens(tok, window=WINDOW)

    before = m.stats.clone()
    fused_cbow()
    torch.cuda.synchronize()
    cbow_targets = int((m.stats - before)[1].item())
    before = m.stats.clone()
    fused_sg()
    torch.cuda.synchronize()
    sg_targets = int((m.stats - before)[1].item())
    kept = int((seq[:n] >= 0).sum())
    torch_targets = int((targets >= 0).sum())
    res["counts"] = dict(tokens=n_tok, kept=kept, cbow_centers=n_live, contexts=n_ctx, cbow_targets=cbow_targets,
                         skipgram_targets=sg_targets, torch_targets=torch_targets, torch_noise_voids=voids)
    paths = {"fused_cbow": fused_cbow, "fused_skipgram": fused_sg, "torch_cbow": torch_cbow,
             "cbow_kernel": lambda: native.w2v_window_fused(*m._w2v_scratch[:3], m.w_in.table_c, m.w_out.table_c,
                                                            LR, window=WINDOW, negative=NEG, vocab=VOCAB,
                                                            seed=m.seed, step=m.step_no, cdf=m._noise_cdf,
                                                            last_nonzero=m._noise_last, cbow=True),
             "subsample": lambda: native.w2v_subsample(tok, VOCAB, m._keep_p, seed=m.seed, step=m.step_no,
                                                       scratch=m._w2v_scratch)}
    for fn in paths.values():      # warm every shape
        fn()
    torch.cuda.synchronize()
    rounds = {k: [] for k in paths}
    for _ in range(a.rounds):
        for k, fn in paths.items():
            rounds[k].append(_events(fn, a.iters))
    row = 4 * m.w_in.stride
    bytes_cbow = (2 * n_ctx + 2 * cbow_targets) * row
    bytes_sg = (2 * kept + 2 * sg_targets) * row
    upd = {"fused_cbow": cbow_targets, "fused_skipgram": sg_targets, "torch_cbow": torch_targets}
    out = {}
    for k, r in rounds.items():
        s = _summary(r)
        med = s["ms_median"] / 1e3
        if k in upd:
            s["words_per_s"] = round(n_tok / med)
            s["target_updates_per_s"] = round(upd[k] / med)
        if k in ("fused_cbow", "cbow_kernel", "torch_cbow"):
            s["tb_per_s_bytes_model"] = round(bytes_cbow / med / 1e12, 3)
        if k == "fused_skipgram":
            s["tb_per_s_bytes_model"] = round(bytes_sg / med / 1e12, 3)
        out[k] = s
    res["ms"] = out
    res["bytes_model"] = dict(row_bytes=row, cbow_bytes=bytes_cbow, skipgram_bytes=bytes_sg,
                              ratio=round(bytes_sg / bytes_cbow, 3))
    res["speedup_cbow_over_torch_cbow"] = round(out["torch_cbow"]["ms_median"] / out["fused_cbow"]["ms_median"], 3)
    res["speedup_cbow_over_skipgram"] = round(out["fused_skipgram"]["ms_median"] / out["fused_cbow"]["ms_median"], 3)
    m.check_finite()
    assert torch.isfinite(W_in).all() and torch.isfinite(W_out).all()
    res["card_after"] = card()
    m.close()
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
