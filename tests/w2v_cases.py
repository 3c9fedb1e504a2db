"""What the skip-gram and CBOW GPU suites of the fused window kernel share: the dispatch rungs, the sweep over them,
the fp32-against-fp64 tolerance, the tables, one direct kernel call and the noise distributions."""
import functools

import numpy as np
import torch

from fps_b200.ops import native

SEED = 4

# fps_w2v_window_fused dispatches on the row stride (the dim rounded up to 4 floats; nvec = stride / 4 float4) to
# fps_w2v_kernel<CBOW, LPR, VPL, MINB, TB>: LPR lanes per row, VPL float4 per lane, MINB CTAs per SM and TB
# target slots (and under CBOW context rows) pulled per block.
#   dim  stride  nvec  <LPR, VPL, MINB, TB>
#     3      4     1   < 1, 1, 2, 8>   padding column 3
#     4      4     1   < 1, 1, 2, 8>
#     8      8     2   < 2, 1, 2, 8>
#    13     16     4   < 4, 1, 2, 8>   padding columns 13-15
#    16     16     4   < 4, 1, 2, 8>
#    24     24     6   < 8, 1, 2, 8>   lanes 6-7 hold nothing
#    36     36     9   <16, 1, 2, 8>   lanes 9-15 hold nothing
#   100    100    25   <32, 1, 2, 8>   lanes 25-31 hold nothing
#   136    136    34   <32, 2, 1, 8>   lanes 0-1 hold 2 float4, the others 1
#   256    256    64   <32, 2, 1, 8>
#   300    300    75   <32, 3, 1, 8>   lanes 0-10 hold 3 float4, the others 2
#   387    388    97   <32, 4, 1, 6>   padding column 387; lane 0 holds 4 float4, the others 3
#   388    388    97   <32, 4, 1, 6>
#   512    512   128   <32, 4, 1, 6>
RUNGS = {3: (1, 1, 8), 4: (1, 1, 8), 8: (2, 1, 8), 13: (4, 1, 8), 16: (4, 1, 8), 24: (8, 1, 8), 36: (16, 1, 8),
         100: (32, 1, 8), 136: (32, 2, 8), 256: (32, 2, 8), 300: (32, 3, 8), 387: (32, 4, 6), 388: (32, 4, 6),
         512: (32, 4, 6)}   # dim -> (LPR, VPL, TB)

SWEEP = [(dim, neg) for dim, (lpr, _, _) in RUNGS.items() for neg in sorted({0, 1, lpr, lpr + 1, 7, 8, 20})]

# The fp32 kernel against the fp64 replay: 2e-5 relative plus 1e-5 of the table's largest value.  The same replay
# run in numpy fp32 stays within a tenth of this at dim 512 with 255 negatives, while a block one slot off or voids
# compacted before blocking move rows by ~1e-3.
RTOL, ATOL_OF_MAX = 2e-5, 1e-5


def close(got, want, what):
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL_OF_MAX * float(np.abs(want).max()), err_msg=what)


def tables(vocab, dim, scale, seed, dev):
    """W_in and W_out ``[vocab, stride]`` fp32, uniform on +-scale, padding columns 0."""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for _ in range(2):
        t = torch.zeros(vocab, (dim + 3) // 4 * 4, device=dev)
        t[:, :dim] = (torch.rand(vocab, dim, generator=g, device=dev) * 2 - 1) * scale
        out.append(t)
    return out


def fused(W_in, W_out, dim, tokens, vocab, *, lr, window, neg, step=0, max_tries=32, cdf=None, last=0, keep_p=None,
          reserve=0, cbow=False):
    """One call through native.w2v_subsample + native.w2v_window_fused; returns (stats, token_stats, nan_flag)."""
    dev = W_in.device
    st = torch.zeros(2, dtype=torch.float32, device=dev)
    ts = torch.zeros(4, dtype=torch.int64, device=dev)
    nan = torch.zeros(1, dtype=torch.int32, device=dev)
    seq, pos, n_comp = native.w2v_subsample(tokens, vocab, keep_p, seed=SEED, step=step, token_stats=ts)
    native.w2v_window_fused(seq, pos, n_comp, native.local_table(W_in, dim), native.local_table(W_out, dim), lr,
                            window=window, negative=neg, vocab=vocab, seed=SEED, step=step, cdf=cdf,
                            last_nonzero=last, max_tries=max_tries, stats=st, token_stats=ts, nan_flag=nan,
                            reserve_total=reserve, cbow=cbow)
    torch.cuda.synchronize()
    return st.cpu(), ts.cpu(), int(nan.item())


VOCAB = 100_000


@functools.lru_cache(maxsize=None)
def noise_dist(kind):
    """(counts, cdf, last_nonzero) of the unigram noise: 30% of the words and the last 1000 have weight 0."""
    if kind == "uniform":
        return None, None, 0
    g = np.random.default_rng(11)
    c = g.integers(1, 50, size=VOCAB).astype(np.float64)
    c[g.random(VOCAB) < 0.3] = 0.0
    c[-1000:] = 0.0
    cdf = native.noise_cdf(torch.from_numpy(c).cuda(), 0.75).cpu().numpy()
    return c, cdf, int(np.flatnonzero(c)[-1])
