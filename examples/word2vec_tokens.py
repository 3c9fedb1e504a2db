#!/usr/bin/env python
"""word2vec skip-gram (or CBOW) from a token stream on one GPU: a seeded topic corpus, frequent-word subsampling,
dynamic windows, linear rate decay (``DeviceSkipGram.fit_tokens``), then nearest neighbours (``most_similar``).

    python examples/word2vec_tokens.py [--vocab 5000 --topics 50 --epochs 3] [--cbow]

``--cbow`` trains CBOW at word2vec.c's CBOW rate 0.05 instead of skip-gram at 0.025.

Word ``w`` of ``topic_corpus`` belongs to topic ``w % topics``, so a neighbour list is right where it shares its
word's topic; the script prints that precision@10 next to the chance level."""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", type=int, default=5000)
    ap.add_argument("--topics", type=int, default=50)
    ap.add_argument("--sentences", type=int, default=60000)
    ap.add_argument("--dim", type=int, default=100)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--cbow", action="store_true", help="train CBOW instead of skip-gram")
    a = ap.parse_args()
    import fps_b200  # noqa: F401
    from fps_b200.models.w2v import DeviceSkipGram
    from fps_b200.utils.synthetic import topic_corpus

    torch.cuda.set_device(0)
    tokens = topic_corpus(a.vocab, a.topics, 12, a.sentences, seed=0)     # sentences separated by -1
    counts = np.bincount(tokens[tokens >= 0].numpy(), minlength=a.vocab)
    m = DeviceSkipGram(a.vocab, a.dim, learning_rate=0.05 if a.cbow else 0.025, negative=5, word_counts=counts, noise_counts=counts,
                       sample=1e-3)
    m.fit_tokens(tokens.pin_memory(), epochs=a.epochs, batch_tokens=1 << 18, window=5, cbow=a.cbow)
    m.check_finite()
    tokens_seen, kept, contexts, dropped = m.token_stats.tolist()
    print(f"{tokens_seen} tokens, {kept} kept after subsampling, {contexts} contexts, {dropped} invalid ids")
    words = torch.arange(a.vocab, device="cuda")
    _, ids = m.most_similar(words, 10)
    prec = ((ids % a.topics) == (words % a.topics)[:, None]).float().mean().item()
    print(f"same-topic precision@10: {prec:.3f} (chance {(a.vocab / a.topics - 1) / (a.vocab - 1):.3f})")
    for w in range(3):
        print(f"word {w}: neighbours {ids[w].tolist()}")
    m.close()


if __name__ == "__main__":
    main()
