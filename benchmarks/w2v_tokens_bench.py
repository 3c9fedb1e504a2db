#!/usr/bin/env python
"""Skip-gram from a token stream: the fused center-window path (``DeviceSkipGram.train_tokens``) against the pair
path (the same pairs expanded in torch, then ``DeviceSkipGram.step``) on one GPU.

    python benchmarks/w2v_tokens_bench.py [--out profiles/h100_w2v_tokens_bench.json]

Shape: 1M words x 300, ``negative=5`` (unigram noise from the corpus counts), ``window=5``, ``sample=1e-3``, a Zipf
``topic_corpus`` (1000 topics, sentences of 20 words) of about 3.1M tokens per call.  Records, in one process:

* the card (name, power limit, max SM clock), before and after;
* per path, ms per call, words per second and target updates per second.  The fused call is its two kernels;
  the pair path is the expansion (torch, from the compacted sequence and the same radii) plus ``step()``
  (the noise sampler and the pointwise kernel), each also timed alone, as is the subsample kernel;
* TB/s by the bytes model (DESIGN §2.13): a fused center moves its ``W_in`` row twice and every target row twice,
  a pair-path record moves both of its rows twice.

The two paths are alternated round by round; the median and the spread over the rounds are kept.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "benchmarks"))

from mf_bpr_bench import card  # noqa: E402

VOCAB, DIM, NEG, WINDOW, SAMPLE = 1_000_000, 300, 5, 5, 1e-3
TOPICS, SENT_LEN, SENTENCES = 1000, 20, 150_000


def _events(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _summary(rounds):
    med = statistics.median(rounds)
    return {"ms_rounds": [round(x, 4) for x in rounds], "ms_median": round(med, 4),
            "ms_spread": round(max(rounds) - min(rounds), 4)}


def _philox_np(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (the kernels' generator), for the radii of the pair path."""
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint32).copy() for x in np.broadcast_arrays(c0, c1, c2, c3))
    k0, k1 = int(k0), int(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0, p1 = M0 * c0.astype(np.uint64), M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), p0.astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), p1.astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint32(k0), lo1, hi0 ^ c3 ^ np.uint32(k1), lo0
            k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def expand_pairs(seq, n, radius):
    """(center, context) pairs of the compacted sequence ``seq[:n]`` with per-entry radii, in torch."""
    s = seq[:n].long()
    seg = torch.cumsum((s < 0).long(), 0)
    idx = torch.arange(n, device=s.device)
    cs, xs = [], []
    for o in list(range(-WINDOW, 0)) + list(range(1, WINDOW + 1)):
        q = (idx + o).clamp(0, n - 1)
        ok = (s >= 0) & (idx + o >= 0) & (idx + o < n) & (s[q] >= 0) & (seg[q] == seg) & (radius >= abs(o))
        cs.append(s[ok]); xs.append(s[q][ok])
    return torch.cat(cs).int(), torch.cat(xs).int()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_w2v_tokens_bench.json"))
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
                                                 topics=TOPICS, sentence_len=SENT_LEN, sentences=SENTENCES)}
    tok_h = topic_corpus(VOCAB, TOPICS, SENT_LEN, SENTENCES, seed=1)
    counts = np.bincount(tok_h[tok_h >= 0].numpy(), minlength=VOCAB).astype(np.float64)
    tok = tok_h.to(dev)
    n_tok = tok.numel()
    m = DeviceSkipGram(VOCAB, DIM, learning_rate=0.025, negative=NEG, seed=1, word_counts=counts,
                       noise_counts=counts, sample=SAMPLE)
    step0 = m.step_no
    # the pair path trains the pairs of the fused path's first call: same compaction, same radii
    seq, pos, n_comp = native.w2v_subsample(tok, VOCAB, m._keep_p, seed=m.seed, step=step0)
    n = int(n_comp.item())
    rad = torch.from_numpy(radii(pos[:n].cpu().numpy(), WINDOW, step0, m.seed, _philox_np)).to(dev)
    centers, contexts = expand_pairs(seq, n, rad)
    n_pairs = centers.numel()
    kept = int((seq[:n] >= 0).sum())
    before = m.stats.clone()
    m.train_tokens(tok, window=WINDOW)
    torch.cuda.synchronize()
    fused_targets = int((m.stats - before)[1].item())
    pair_records = n_pairs * (1 + NEG)
    res["counts"] = dict(tokens=n_tok, kept=kept, pairs=n_pairs, fused_targets=fused_targets,
                         pair_records=pair_records)

    def fused():
        m.train_tokens(tok, window=WINDOW)

    def pair():
        c, x = expand_pairs(seq, n, rad)
        m.step(c, x)

    parts = {"subsample": lambda: native.w2v_subsample(tok, VOCAB, m._keep_p, seed=m.seed, step=m.step_no,
                                                       scratch=m._w2v_scratch),
             "window_kernel": lambda: native.w2v_window_fused(*m._w2v_scratch[:3], m.w_in.table_c, m.w_out.table_c,
                                                              m.lr, window=WINDOW, negative=NEG, vocab=VOCAB,
                                                              seed=m.seed, step=m.step_no, cdf=m._noise_cdf,
                                                              last_nonzero=m._noise_last),
             "pair_expansion": lambda: expand_pairs(seq, n, rad),
             "pair_step": lambda: m.step(centers, contexts)}
    for fn in (fused, pair, *parts.values()):      # warm every shape
        fn()
    torch.cuda.synchronize()
    rounds = {k: [] for k in ("fused", "pair", *parts)}
    for _ in range(a.rounds):
        rounds["fused"].append(_events(fused, a.iters))
        rounds["pair"].append(_events(pair, a.iters))
        for k, fn in parts.items():
            rounds[k].append(_events(fn, a.iters))
    row = 4 * m.w_in.stride
    bytes_fused = (2 * kept + 2 * fused_targets) * row
    bytes_pair = 4 * pair_records * row
    out = {}
    for k, r in rounds.items():
        s = _summary(r)
        med = s["ms_median"] / 1e3
        if k in ("fused", "pair"):
            s["words_per_s"] = round(n_tok / med)
            s["target_updates_per_s"] = round((fused_targets if k == "fused" else pair_records) / med)
        if k == "window_kernel":
            s["tb_per_s_bytes_model"] = round(bytes_fused / med / 1e12, 3)
        if k == "pair_step":
            s["tb_per_s_bytes_model"] = round(bytes_pair / med / 1e12, 3)
        out[k] = s
    res["ms"] = out
    res["bytes_model"] = dict(row_bytes=row, fused_bytes=bytes_fused, pair_bytes=bytes_pair,
                              ratio=round(bytes_pair / bytes_fused, 3))
    res["speedup_fused_over_pair"] = round(out["pair"]["ms_median"] / out["fused"]["ms_median"], 3)
    m.check_finite()
    res["card_after"] = card()
    m.close()
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
