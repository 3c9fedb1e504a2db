"""Host side of the device top-K seen-item exclusion: the per-user window state that builds the
exclusion lists, and the normalisation of an exclusion CSR (plain torch ops, run here on CPU tensors)."""
import numpy as np
import pytest
import torch


def _stream(seed, n_users=6, n_items=12, n_runs=40):
    """Ratings in runs of one user (so batch boundaries can fall inside a run), items drawn from a small
    pool so that items repeat inside a user's window."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n_runs):
        u = int(rng.randint(n_users))
        for _ in range(int(rng.randint(1, 5))):
            out.append((u, int(rng.randint(n_items))))
    return out


def _sets_of_seen_filter(stream, memory, n_items):
    """The set ``_seen_filter`` excludes for every rating: give it every item as a candidate."""
    from fps_b200.models.mf.device_api import _seen_filter

    everything = [(0.0, i) for i in range(n_items)]
    rows = [(u, i, t, everything) for t, (u, i) in enumerate(stream)]
    return [set(range(n_items)) - {i for _, i in kept}
            for (_u, _i, _t, kept) in _seen_filter(rows, n_items, memory)]


def _boundaries(stream, how):
    n = len(stream)
    if how == "runs":             # cut exactly between runs of a user
        return [0] + [j for j in range(1, n) if stream[j][0] != stream[j - 1][0]] + [n]
    if how == "inside":           # cut after the first rating of every run (inside the run)
        cuts = [j + 1 for j in range(n - 1) if j == 0 or stream[j][0] != stream[j - 1][0]]
        return sorted(set([0] + cuts + [n]))
    step = int(how)
    return list(range(0, n, step)) + [n]


@pytest.mark.parametrize("memory", [0, 1, 2, 5, -1])
@pytest.mark.parametrize("how", ["1", "7", "runs", "inside"])
def test_seen_window_matches_seen_filter(memory, how):
    from fps_b200.models.mf.device_api import _SeenWindow

    n_items = 12
    for seed in range(3):
        stream = _stream(seed + 10 * (memory + 1), n_items=n_items)
        want = _sets_of_seen_filter(stream, memory, n_items)
        w = _SeenWindow(memory)
        got = []
        cuts = _boundaries(stream, how)
        for a, b in zip(cuts[:-1], cuts[1:]):
            batch = stream[a:b]
            off, ids = w.exclusions([u for u, _ in batch], [i for _, i in batch])
            assert off.dtype == np.int64 and ids.dtype == np.int64
            assert off.shape == (len(batch) + 1,) and off[0] == 0 and off[-1] == ids.size
            for j in range(len(batch)):
                part = ids[off[j]:off[j + 1]].tolist()
                assert len(part) == len(set(part))
                got.append(set(part))
        assert got == want
        if memory == 0:
            assert all(not s for s in got)


def test_seen_window_keeps_the_repeat_quirk():
    """An item rated twice inside the window leaves the set when its OLDER copy leaves the window."""
    from fps_b200.models.mf.device_api import _SeenWindow

    w = _SeenWindow(2)
    off, ids = w.exclusions([0, 0, 0, 0], [5, 5, 7, 8])
    sets = [set(ids[off[j]:off[j + 1]].tolist()) for j in range(4)]
    # rating 3 pushes the first 5 out of the window and takes 5 out of the set, although the second 5
    # is still inside the window: rating 4 excludes only {7}
    assert sets == [set(), {5}, {5}, {7}]
    off, ids = w.exclusions([0], [9])
    assert set(ids.tolist()) == {7, 8}


def _reference_normalize(offsets, rows, n_q, n_items, inv_perm):
    out = []
    for q in range(n_q):
        vals = {int(r) for r in rows[offsets[q]:offsets[q + 1]] if 0 <= int(r) < n_items}
        if inv_perm is not None:
            vals = {int(inv_perm[r]) for r in vals}
        out.append(sorted(vals))
    return out


@pytest.mark.parametrize("with_perm", [False, True])
def test_normalize_exclude_on_cpu(with_perm):
    from fps_b200.models.mf.device_topk import normalize_exclude

    g = torch.Generator().manual_seed(5)
    n_q, n_items = 9, 50
    lens = torch.randint(0, 12, (n_q,), generator=g)
    lens[3] = 0                                                  # empty row
    offsets = torch.zeros(n_q + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(lens, 0)
    rows = torch.randint(-5, n_items + 5, (int(offsets[-1]),), generator=g)   # out-of-range values
    rows[:4] = rows[0]                                           # duplicates inside a row
    perm = torch.randperm(n_items, generator=g) if with_perm else None
    inv_perm = None
    if perm is not None:
        inv_perm = torch.empty_like(perm)
        inv_perm[perm] = torch.arange(n_items)
    off, pos, cnt = normalize_exclude(offsets, rows, n_q, n_items, inv_perm)
    assert off.dtype == pos.dtype == cnt.dtype == torch.int32
    want = _reference_normalize(offsets.tolist(), rows.tolist(), n_q, n_items,
                                inv_perm.tolist() if inv_perm is not None else None)
    assert cnt.tolist() == [len(w) for w in want]
    assert off[0] == 0 and off.tolist()[1:] == np.cumsum([len(w) for w in want]).tolist()
    for q in range(n_q):
        assert pos[off[q]:off[q + 1]].tolist() == want[q]
    # int32 inputs and a row list longer than offsets[-1] (the tail belongs to no query)
    off2, pos2, cnt2 = normalize_exclude(offsets.to(torch.int32), torch.cat([rows, torch.tensor([1, 2])]).to(torch.int32),
                                         n_q, n_items, inv_perm)
    assert torch.equal(off2, off) and torch.equal(pos2, pos) and torch.equal(cnt2, cnt)
    with pytest.raises(ValueError):
        normalize_exclude(offsets[:-1], rows, n_q, n_items)
