"""Device top-K recommendation (K6 / K12): pull query vectors from the PS, score them against the
worker-local item table on the Hopper tensor cores (wgmma), keep an exact top-K.

Capability of ``psTopKGenerator`` / the generator half of ``psOnlineLearnerAndGenerator``
(PSTopKGenerator.scala:47-107, PSTopKGeneratorWorker.scala:35-114): user vectors live on the PS,
item vectors on the workers, every query is answered by every worker with its local top-``workerK``
and the partial lists are merged (``merge_partial_topk`` = CollectTopKFromEachWorker).

Algorithm (exact, tile-pruned -- the GPU-idiomatic replacement of the LEMP bucket scan):
  pass 1  tensor-core GEMM, epilogue keeps only the per-(query, 128-item tile) maximum;
  theta   K-th largest tile maximum per query  (a lower bound of the true K-th best score);
  pass 2  same GEMM, epilogue appends every (score, item) >= theta  (a few x K candidates);
  select  top-K of the candidates.
Scores are TF32 products accumulated in FP32; ``rescore=True`` recomputes the K winners in full
FP32 (ordering among near-ties may then differ from the TF32 ranking by < 1e-3 relative).
Rows may be up to ``native.TOPK_MAX_STRIDE`` = 512 floats wide; above 128 the scoring kernel streams
the item table by 32-float K block (same passes, same exactness).

Per-query exclusion (``topk(..., exclude=...)``, the seen-item filter of CollectTopKFromEachWorker):
let ``E_q`` be the number of distinct excluded items of query ``q`` present in the table.  The
``(K + E_q)``-th largest tile maximum is still a lower bound of the K-th best *admissible* score:
those ``K + E_q`` tiles hold ``K + E_q`` distinct items scoring at least that much, and at most ``E_q``
of them are excluded.  The same argument holds for the LENGTH-pruned ``theta0`` (prefix of the
table) and for the overflow tightening (the ``(K + E_q)``-th best kept candidate); the tile count of
``_tiles_needed`` follows from theta unchanged.  When ``K + E_q`` exceeds the tiles scored, theta is
-3e38: the row overflows into the brute-force fallback (excluded columns masked), so the result stays
exact.  Excluded candidates are dropped in the select stage (``fps_row_topk``); the scoring kernel
is not involved.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from ...ops import native
from ...store.sharded_table import ShardedTable


def normalize_exclude(offsets, rows, n_q: int, n_items: int, inv_perm: Optional[torch.Tensor] = None,
                      device=None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Per-query exclusion CSR in the caller's row numbering -> the form ``fps_row_topk`` reads.

    ``offsets`` [n_q + 1] and ``rows`` may be unsorted within a query and hold duplicates or values
    outside ``[0, n_items)`` (ignored).  Rows are mapped through ``inv_perm`` (caller row -> table
    position) when given, then sorted and de-duplicated per query with one sort on ``query * n_items +
    position`` keys.  Returns ``(offsets int32 [n_q + 1], positions int32 [E], counts int32 [n_q])`` on
    ``device`` (default: the device of ``rows``).  Plain torch ops, no host loop."""
    dev = torch.device(device) if device is not None else torch.as_tensor(rows).device
    off = torch.as_tensor(offsets).to(dev, torch.int64).reshape(-1)
    r = torch.as_tensor(rows).to(dev, torch.int64).reshape(-1)
    if off.numel() != n_q + 1:
        raise ValueError(f"exclude offsets must have n_q + 1 = {n_q + 1} entries, got {off.numel()}")
    j = torch.arange(r.numel(), device=dev)
    q = torch.searchsorted(off[1:].contiguous(), j, right=True)        # query of entry j
    keep = (j >= off[0]) & (q < n_q) & (r >= 0) & (r < n_items)
    q, r = q[keep], r[keep]
    if inv_perm is not None:
        r = inv_perm[r]
    key = torch.unique_consecutive(torch.sort(q * n_items + r).values)
    cnt = torch.bincount(key // n_items, minlength=n_q)
    out_off = torch.zeros(n_q + 1, dtype=torch.int64, device=dev)
    out_off[1:] = torch.cumsum(cnt, 0)
    return out_off.to(torch.int32), (key % n_items).to(torch.int32), cnt.to(torch.int32)


class DeviceTopK:
    """``sort_by_length=True`` adds the LEMP LENGTH bound at tile granularity (K6;
    LEMPPruningFunctions.scala:20-27, the bucket early-exit of PSTopKGeneratorWorker.scala:86-90): the
    item table is kept sorted by vector length (descending), so every 128-item tile has a known
    maximum length and a tile can contain a top-K item of query ``q`` only if
    ``maxLen(tile) * |q| >= theta_q``.  The tiles that survive form a *prefix* of the table, so pruning
    is simply running the same tensor-core kernel over fewer rows -- no pointer chasing."""

    LENGTH_SLACK = 1.004  # TF32 products may exceed the fp32 Cauchy-Schwarz bound by ~2^-10 relative

    def __init__(self, items: torch.Tensor, max_batch_bytes: int = 512 << 20, sort_by_length: bool = False,
                 pass1_fraction: Optional[float] = None):
        if items.dim() != 2 or items.shape[1] % 4 != 0:
            raise ValueError("items must be [n_items, stride] with stride % 4 == 0")
        native.check_topk_stride(items.shape[1])
        self.perm = self.inv_perm = None
        if sort_by_length:
            lens = items.norm(dim=1)
            self.perm = torch.argsort(lens, descending=True)
            self.inv_perm = torch.empty_like(self.perm)
            self.inv_perm[self.perm] = torch.arange(self.perm.numel(), device=self.perm.device)
            items = items[self.perm].contiguous()
            self.tile_maxlen = lens[self.perm][:: native.TOPK_TILE].contiguous()
        self.items = items
        self.n_items, self.stride = items.shape
        self.n_tiles = (self.n_items + native.TOPK_TILE - 1) // native.TOPK_TILE
        self.max_batch_bytes = max_batch_bytes
        # theta is computed from the first `pass1_fraction` of the tiles only: the K-th largest tile maximum
        # of ANY subset of tiles is still a valid lower bound (K distinct items reach it), just a weaker
        # one -- pass 1 shrinks to that fraction, pass 2 keeps a few more candidates (identical results).
        # 1/8 is the default for tables of >= 512 tiles (0 / None: scan every tile in pass 1).
        if pass1_fraction is None:
            pass1_fraction = 0.125 if self.n_tiles >= 512 else 0.0
        self.pass1_fraction = pass1_fraction
        self._last = (0, None, None)
        self.last_fallback_rows = 0       # rows the last ``topk`` answered by brute force (overflow)
        self.trace = None                 # set to [] to collect (stage, ms) pairs (synchronising!)
        self._t0 = None

    def _mark(self, label: str) -> None:
        if self.trace is None:
            return
        import time
        torch.cuda.synchronize()
        now = time.perf_counter()
        if self._t0 is not None:
            self.trace.append((label, (now - self._t0) * 1e3))
        self._t0 = now

    def _tiles_needed(self, theta: torch.Tensor, qnorm: torch.Tensor) -> torch.Tensor:
        """int32 device scalar: number of leading tiles (of the length-sorted table) that can still hold
        a score >= theta for at least one query of the batch.  Stays on the device: the scoring kernel
        reads it as its tile limit, so pruning costs no host round trip."""
        bound = torch.where((theta > 0) & (qnorm > 0), theta / qnorm.clamp_min(1e-30),
                            torch.full_like(theta, -1.0))          # theta <= 0: the bound cannot prune
        # the batch needs the prefix of its least selective query; tile_maxlen is descending
        return (self.tile_maxlen * self.LENGTH_SLACK >= bound.min()).sum().to(torch.int32).reshape(1)

    @property
    def last_tiles_scored(self) -> Tuple[int, int]:
        """(pass 1, pass 2) tiles scored by the last ``topk`` chunk (synchronises)."""
        p1, lim1, lim2 = self._last
        t1 = p1 if lim1 is None else max(p1, min(self.n_tiles, int(lim1.item())))
        t2 = self.n_tiles if lim2 is None else min(self.n_tiles, int(lim2.item()))
        return t1, t2

    # -- raw scores (validation / tiny problems) ---------------------------------------------
    def scores(self, *, q_ids=None, q_table: Optional[ShardedTable] = None, q_local=None) -> torch.Tensor:
        """[n_q, n_items] scores in the caller's item order."""
        n_q = q_ids.numel() if q_ids is not None else q_local.shape[0]
        out = torch.empty((n_q, self.n_items), dtype=torch.float32, device=self.items.device)
        native.topk_mma(self.items, 0, q_ids=q_ids, q_tab=q_table.table_c if q_table else None,
                        q_local=q_local, out_scores=out)
        if self.perm is not None:
            unsorted = torch.empty_like(out)
            unsorted[:, self.perm] = out
            out = unsorted
        return out

    def topk(self, K: int, *, q_ids=None, q_table: Optional[ShardedTable] = None, q_local=None,
             rescore: bool = False, exclude=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Returns ``(scores [n_q, K'], item_rows [n_q, K'])`` best first, ``K' = min(K, n_items)``;
        item_rows index the caller's item table.

        ``exclude=(offsets, rows)``: items query ``q`` must not get, ``rows[offsets[q]:offsets[q+1]]``
        in the caller's row numbering (see :func:`normalize_exclude`).  The result is the exact top-K
        of the remaining items; a query with fewer than ``K'`` of them gets ``(-3e38, -1)`` entries at
        the end."""
        n_q = q_ids.numel() if q_ids is not None else q_local.shape[0]
        Kp = min(K, self.n_items)
        if Kp > 2048:
            raise ValueError("DeviceTopK supports K <= 2048 (shared-memory sort buffer of fps_row_topk)")
        T = native.TOPK_TILE
        dev = self.items.device
        ex = None
        Ke = Kp                              # K plus the largest per-query exclusion count
        if exclude is not None:
            ex_off, ex_pos, ex_cnt = normalize_exclude(exclude[0], exclude[1], n_q, self.n_items,
                                                       self.inv_perm, device=dev)
            if ex_pos.numel() > 0:
                host = torch.cat([ex_off, ex_cnt.max().reshape(1)]).cpu()    # one transfer: offsets + max E_q
                ex = host[:-1]
                Ke = Kp + int(host[-1])
        # candidate buffer: a few x K per query is typical (worst case K*128 and more with ties); an
        # overflowing row raises its theta and repeats pass 2 instead of growing the buffer
        cap = min(max(2048, 16 * Ke), max(T, (self.n_items + T - 1) // T * T) * 2)
        per_row = self.n_tiles * 4 + cap * 8
        chunk = max(256, (self.max_batch_bytes // per_row) // 256 * 256)
        tab = q_table.table_c if q_table is not None else None
        outs, outi = [], []
        self.last_fallback_rows = 0
        for a in range(0, n_q, chunk):
            b = min(n_q, a + chunk)
            ids = q_ids[a:b].contiguous() if q_ids is not None else None
            ql = q_local[a:b].contiguous() if q_local is not None else None
            n = b - a
            kq = c_ex = None                 # per-query K + E_q, and the chunk's exclusion CSR
            if ex is not None:
                e0, e1 = int(ex[a]), int(ex[b])
                c_ex = ((ex_off[a:b + 1] - e0).contiguous(), ex_pos[e0:e1])
                kq = (ex_cnt[a:b] + Kp).contiguous()
            self._mark("start")
            kw = dict(q_ids=ids, q_tab=tab, q_local=ql)
            # ---- pass 1: per-(query, tile) maxima ------------------------------------------------
            lim1 = lim2 = None
            p1 = self.n_tiles
            prune = self.perm is not None and self.n_tiles >= 16 and max(Ke, self.n_tiles // 8) < self.n_tiles
            frac_tiles = 0
            if not prune and self.pass1_fraction:
                frac_tiles = max(Ke, int(self.n_tiles * float(self.pass1_fraction)))
            if not prune and 0 < frac_tiles < self.n_tiles:
                p1 = frac_tiles
                tile_max = torch.full((n, self.n_tiles), -3.0e38, dtype=torch.float32, device=dev)
                first = torch.full((1,), p1, dtype=torch.int32, device=dev)
                native.topk_mma(self.items, 1, tile_max=tile_max, tile_limit=first, **kw)
                self._mark("pass1-prefix")
            elif not prune:
                tile_max = torch.empty((n, self.n_tiles), dtype=torch.float32, device=dev)
                native.topk_mma(self.items, 1, tile_max=tile_max, **kw)
                self._mark("pass1")
            else:
                # LENGTH-pruned pass 1: score the tiles of the longest items first; their K-th best tile
                # maximum already bounds how far down the length-sorted table a top-K item can sit.
                q = q_table.pull(ids) if ids is not None else ql
                qnorm = q.norm(dim=1)
                p1 = max(Ke, self.n_tiles // 8)
                tile_max = torch.full((n, self.n_tiles), -3.0e38, dtype=torch.float32, device=dev)
                first = torch.full((1,), p1, dtype=torch.int32, device=dev)
                native.topk_mma(self.items, 1, tile_max=tile_max, tile_limit=first, **kw)
                self._mark("pass1a")
                theta0 = native.row_kth_largest(tile_max, Kp, n_cols=p1, k_per_row=kq)
                lim1 = self._tiles_needed(theta0, qnorm)
                native.topk_mma(self.items, 1, tile_max=tile_max, tile_lo=p1, tile_limit=lim1, **kw)
                self._mark("pass1b")
            theta = native.row_kth_largest(tile_max, Kp, k_per_row=kq)  # -3e38 with fewer than K (+E_q) tiles
            if prune:
                lim2 = self._tiles_needed(theta, qnorm)       # <= tiles scored in pass 1 (theta >= theta0)
            self._mark("theta")
            # ---- pass 2: candidates >= theta, progressive tightening on overflow ---------------
            _, n_splits, seg_cap = native.topk_geometry(self.items, n, 0, cap)
            cnt = torch.empty((n, n_splits), dtype=torch.int32, device=dev)
            cs = torch.empty((n, cap), dtype=torch.float32, device=dev)
            ci = torch.zeros((n, cap), dtype=torch.int32, device=dev)
            bad = None
            for attempt in range(4):
                cs.fill_(-3.0e38)                               # unused slots of a segment never win
                native.topk_mma(self.items, 2, theta=theta, cand_count=cnt, cand_score=cs, cand_item=ci,
                                tile_limit=lim2, **kw)
                over = (cnt > seg_cap).any(dim=1)
                self._mark("pass2")
                if not bool(over.any().item()):                 # the one host sync of the pipeline
                    break
                if attempt == 3:
                    bad = torch.nonzero(over).flatten()
                    break
                # K-th best of the candidates that were kept: a valid, higher lower bound
                theta = torch.maximum(theta, native.row_kth_largest(cs, Kp, k_per_row=kq))
                if prune:
                    lim2 = torch.minimum(lim2, self._tiles_needed(theta, qnorm))
                self._mark("tighten")
            self._last = (p1, lim1, lim2)
            sc, rows = native.row_topk(cs, ci, Kp, exclude=c_ex)  # select + sort, one CTA per row
            self._mark("select")
            rows = rows.to(torch.int64)
            if bad is not None:
                # rows that still overflow (e.g. thousands of items tied at theta, an all-zero query):
                # brute force, always exact
                self.last_fallback_rows += bad.numel()
                bq = dict(q_ids=ids[bad].contiguous(), q_tab=tab) if ids is not None else \
                    dict(q_local=ql[bad].contiguous())
                for s0 in range(0, bad.numel(), 64):
                    sel = bad[s0:s0 + 64]
                    full = torch.empty((sel.numel(), self.n_items), dtype=torch.float32, device=dev)
                    sub = {k: (v[s0:s0 + 64].contiguous() if torch.is_tensor(v) else v) for k, v in bq.items()}
                    native.topk_mma(self.items, 0, out_scores=full, **sub)
                    if c_ex is not None:
                        _mask_excluded(full, sel, n, *c_ex)
                    top = torch.topk(full, Kp, dim=1)
                    sc[sel], rows[sel] = top.values, top.indices
            if c_ex is not None:
                # fewer than K admissible items: unused candidate slots / masked columns won
                short = sc < -1.0e38
                sc, rows = sc.masked_fill(short, -3.0e38), rows.masked_fill(short, -1)
            if rescore:
                q = (q_table.pull(ids) if ids is not None else ql[:, : self.stride])
                q = torch.nn.functional.pad(q, (0, self.stride - q.shape[1]))
                if c_ex is None:
                    exact = torch.einsum("qd,qkd->qk", q, self.items[rows])
                else:
                    exact = torch.einsum("qd,qkd->qk", q, self.items[rows.clamp_min(0)])
                    exact = exact.masked_fill(rows < 0, -3.0e38)
                order = torch.argsort(exact, dim=1, descending=True)
                sc, rows = torch.gather(exact, 1, order), torch.gather(rows, 1, order)
            if self.perm is not None:       # back to row numbers of the caller's (unsorted) table
                rows = self.perm[rows] if c_ex is None else \
                    torch.where(rows >= 0, self.perm[rows.clamp_min(0)], rows)
            outs.append(sc); outi.append(rows)
        return torch.cat(outs), torch.cat(outi)


def _mask_excluded(full: torch.Tensor, sel: torch.Tensor, n: int, off: torch.Tensor, pos: torch.Tensor) -> None:
    """Brute-force fallback: set the excluded columns of the chunk rows ``sel`` (rows of ``full``) to
    -inf.  ``off`` / ``pos``: the chunk's exclusion CSR over ``n`` rows, table positions."""
    q = torch.repeat_interleave(torch.arange(n, device=full.device), (off[1:] - off[:-1]).long(),
                                output_size=pos.numel())
    slot = torch.full((n,), -1, dtype=torch.int64, device=full.device)
    slot[sel] = torch.arange(sel.numel(), device=full.device)
    m = slot[q]
    hit = m >= 0
    full[m[hit], pos[hit].long()] = float("-inf")


def merge_partial_topk(scores: torch.Tensor, items: torch.Tensor, K: int,
                       seen_mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """K-way merge of per-worker partial lists ``[n_q, W*workerK]`` with an optional seen-item filter
    (CollectTopKFromEachWorker.scala:41-56)."""
    if seen_mask is not None:
        scores = torch.where(seen_mask, torch.full_like(scores, -3.0e38), scores)
    Kp = min(K, scores.shape[1])
    if scores.is_cuda and Kp <= 2048:
        # device K-way merge (K12): select + sort in one kernel; it returns column positions so that
        # item ids of any integer width can be gathered afterwards
        n, C = scores.shape
        pos = torch.arange(C, dtype=torch.int32, device=scores.device).expand(n, C).contiguous()
        sc, where = native.row_topk(scores.contiguous().float(), pos, Kp)
        return sc, torch.gather(items, 1, where.to(torch.int64))
    top = torch.topk(scores, Kp, dim=1)
    return top.values, torch.gather(items, 1, top.indices)


class DistributedTopK:
    """Top-K serving across ranks (capability of ``psTopKGenerator``): user vectors on the PS
    (``user_table``), every rank holds a partition of the items (``local_items`` with their global ids
    ``local_item_ids``); every query is answered by every rank with its local top-``workerK`` (the
    reference broadcasts each rating to all workers, PSTopKGenerator.scala:78-89) and the partial lists
    are merged (E9: gather + K-way merge = ``CollectTopKFromEachWorker``)."""

    def __init__(self, user_table: ShardedTable, local_items: torch.Tensor, local_item_ids: torch.Tensor,
                 group=None):
        import torch.distributed as dist

        self.users, self.group = user_table, group
        self.local = DeviceTopK(local_items)
        self.item_ids = local_item_ids.to(torch.int64)
        self._ids_sorted, self._ids_order = torch.sort(self.item_ids)   # global id -> local row lookup
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1

    def _gather_lists(self, sc: torch.Tensor, gids: torch.Tensor, dst):
        """Partial lists -> the merging rank(s) by one-sided stores into their receive slots
        (:class:`~fps_b200.parallel.fabric.P2PGather`): no NCCL collective on this path."""
        from ..._p2p import gather_pair

        return gather_pair(self, sc, gids, dst, self.group, self.users.device)

    def topk(self, query_user_ids: torch.Tensor, K: int, workerK: Optional[int] = None, dst=None,
             exclude=None):
        """``dst=None``: every rank gets the merged lists; ``dst=r``: only rank ``r`` merges (the
        parallelism-1 sink of CollectTopKFromEachWorker.scala:41-56), the others return ``(None, None)``.
        ``exclude=(offsets, ids)``: per-query CSR of **global item ids** no list may contain; every rank
        drops the ids it does not own, so each partial list is already filtered and the merge is the
        plain one.  Lists with fewer admissible items than ``K`` end in ``(-3e38, -1)`` entries."""
        wk = min(workerK or K, self.local.n_items)
        ex = None
        if exclude is not None:
            g = torch.as_tensor(exclude[1]).to(self.item_ids.device, torch.int64).reshape(-1)
            at = torch.searchsorted(self._ids_sorted, g).clamp_max(self._ids_sorted.numel() - 1)
            ex = (exclude[0], torch.where(self._ids_sorted[at] == g, self._ids_order[at], -1))
        sc, rows = self.local.topk(wk, q_ids=query_user_ids, q_table=self.users, exclude=ex)
        gids = self.item_ids[rows] if ex is None else \
            torch.where(rows >= 0, self.item_ids[rows.clamp_min(0)], -1)
        if self.world == 1:
            return merge_partial_topk(sc, gids, K)
        if wk < (workerK or K):  # pad so all ranks contribute equally sized lists
            pad = (workerK or K) - wk
            sc = torch.nn.functional.pad(sc, (0, pad), value=-3.0e38)
            gids = torch.nn.functional.pad(gids, (0, pad), value=-1)
        got = self._gather_lists(sc.contiguous(), gids.contiguous(), dst)
        if got is None:
            return None, None
        all_sc, all_id = got
        return merge_partial_topk(torch.cat(all_sc, 1), torch.cat(all_id, 1), K)
