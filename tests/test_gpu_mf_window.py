"""The step window of DeviceOnlineMF (fps_mf_window.cu): deferred micro-batches applied item-major in one launch
give the tables of one fused launch per micro-batch, bitwise, and every read sees them applied."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

USERS, ITEMS = 6_000, 1_500


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _pair(k=64, err_mode=1, lr=0.05, users=USERS, items=ITEMS):
    from fps_b200.models.mf.device import DeviceOnlineMF

    kw = dict(learning_rate=lr, seed=11, err_mode=err_mode, range_min=-0.1, range_max=0.1)
    win = DeviceOnlineMF(users, items, k, step_window=8, **kw)
    ref = DeviceOnlineMF(users, items, k, step_window=0, **kw)
    assert win.step_window == 8 and ref.step_window == 0
    return win, ref


def _batch(g, dev, n, users, items, packed, user_pool=None, distinct_items=True):
    from fps_b200.ops import native

    u = user_pool if user_pool is not None else torch.randperm(users, generator=g)[:n]
    i = torch.randperm(items, generator=g)[:n] if distinct_items else torch.randint(0, items, (n,), generator=g)
    r = torch.rand(n, generator=g).half().float()
    u, i = u.int(), i.int()
    if packed:
        return (native.pack_ratings(u, i, r).to(dev),)
    return u.to(dev), i.to(dev), r.to(dev)


def _conflict_free_steps(g, dev, n_steps, per_step, n, packed):
    """Steps of `per_step` micro-batches: distinct users in a step, distinct items in a micro-batch."""
    out = []
    for _ in range(n_steps):
        users = torch.randperm(USERS, generator=g)[: per_step * n].split(n)
        out.append([_batch(g, dev, n, USERS, ITEMS, packed, user_pool=users[j]) for j in range(per_step)])
    return out


def _same_tables(win, ref):
    assert torch.equal(win.users, ref.users)
    assert torch.equal(win.items.local, ref.items.local)


def _same_stats(win, ref):
    a, b = win.stats.double().cpu(), ref.stats.double().cpu()
    assert a[1].item() == b[1].item()
    assert torch.allclose(a[0], b[0], rtol=1e-5)


@pytest.mark.parametrize("k", [16, 64, 128])
@pytest.mark.parametrize("packed", [True, False])
@pytest.mark.parametrize("err_mode", [0, 1])
def test_conflict_free_windows_are_bitwise(dev, k, packed, err_mode):
    win, ref = _pair(k=k, err_mode=err_mode)
    g = torch.Generator().manual_seed(k * 10 + err_mode)
    for step in _conflict_free_steps(g, dev, 6, 5, 1_000, packed):
        for b in step:
            win.step(*b)
            ref.step(*b)
    _same_tables(win, ref)
    _same_stats(win, ref)
    win.close(); ref.close()


def test_users_repeated_across_micro_batches_split_the_window(dev):
    win, ref = _pair()
    g = torch.Generator().manual_seed(3)
    pool = torch.randperm(USERS, generator=g)[:1_200]
    for s in range(12):          # users drawn from a small pool: most micro-batches repeat an earlier user
        users = pool[torch.randperm(1_200, generator=g)[:1_000]]
        b = _batch(g, dev, 1_000, USERS, ITEMS, packed=s % 2 == 0, user_pool=users)
        win.step(*b)
        ref.step(*b)
    _same_tables(win, ref)
    _same_stats(win, ref)


def test_duplicates_inside_a_micro_batch_stay_close(dev):
    win, ref = _pair(lr=0.01)
    g = torch.Generator().manual_seed(4)
    for s in range(10):
        dup = s % 3 == 1        # every third micro-batch repeats items (and users) inside itself
        users = torch.randint(0, USERS, (1_000,), generator=g) if dup else torch.randperm(USERS, generator=g)[:1_000]
        b = _batch(g, dev, 1_000, USERS, ITEMS, packed=False, user_pool=users, distinct_items=not dup)
        win.step(*b)
        ref.step(*b)
    # racy in both paths: an update's delta depends on whether its pull saw a concurrent push to the same row
    # (|lr * e * delta v| ~ 1e-6 per race here), so the tables agree to that, not bitwise
    torch.testing.assert_close(win.users, ref.users, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(win.items.local, ref.items.local, rtol=1e-5, atol=1e-4)
    assert win.stats[1].item() == ref.stats[1].item() == 10_000


def test_more_micro_batches_than_the_window_without_a_read(dev):
    from fps_b200.ops import native

    win, ref = _pair()
    g = torch.Generator().manual_seed(5)
    users = torch.randperm(USERS, generator=g)[:20 * 250].split(250)   # no user twice in 20 micro-batches
    before = native.launch_count()
    for j in range(20):
        b = _batch(g, dev, 250, USERS, ITEMS, packed=True, user_pool=users[j])
        win.step(*b)
        ref.step(*b)
    assert native.launch_count() - before == 20 + 2      # the reference's 20 launches + two full windows
    assert len(win._pending) == 4
    _same_tables(win, ref)
    _same_stats(win, ref)


def test_ineligible_step_between_windowed_ones_keeps_order(dev):
    win, ref = _pair()
    g = torch.Generator().manual_seed(6)
    for s in range(9):
        users = torch.randperm(USERS, generator=g)[:1_000]
        b = _batch(g, dev, 1_000, USERS, ITEMS, packed=False, user_pool=users)
        if s in (3, 7):                          # int64 ids: the per-launch path
            b = (b[0].long(), b[1].long(), b[2])
        win.step(*b)
        ref.step(*b)
        if s in (3, 7):
            assert not win._pending
    _same_tables(win, ref)
    _same_stats(win, ref)


def test_caller_may_reuse_its_tensors(dev):
    win, ref = _pair()
    g = torch.Generator().manual_seed(7)
    steps = _conflict_free_steps(g, dev, 2, 4, 800, packed=False)
    buf = [torch.empty_like(t) for t in steps[0][0]]
    for step in steps:
        for b in step:
            for d, s in zip(buf, b):
                d.copy_(s)
            win.step(*buf)
            for d in buf:
                d.fill_(-7 if d.dtype == torch.int32 else 1e30)   # overwritten right after step()
            ref.step(*b)
    _same_tables(win, ref)


def test_every_read_point_sees_the_window_applied(dev, tmp_path):
    from fps_b200.errors import FactorIsNotANumberException

    g = torch.Generator().manual_seed(8)
    reads = {
        "stats": lambda m: m.stats.clone(),
        "users": lambda m: m.users.clone(),
        "items": lambda m: m.items.local.clone(),
        "nan_flag": lambda m: m.nan_flag.clone(),
        "flush": lambda m: (m.flush(), m._users.clone())[1],
        "predict": lambda m: m.predict(torch.arange(50, device=dev, dtype=torch.int32),
                                       torch.arange(50, device=dev, dtype=torch.int32)),
        "user_vectors": lambda m: m.user_vectors()[1],
        "item_vectors": lambda m: m.item_vectors()[1],
        "check_finite": lambda m: (m.check_finite(), m._users.clone())[1],
        "barrier": lambda m: (m.barrier(), m._users.clone())[1],
        "refresh": lambda m: (m.refresh(), m._items.local.clone())[1],
    }
    for name, read in reads.items():
        win, ref = _pair()
        for b in _conflict_free_steps(g, dev, 1, 3, 500, packed=True)[0]:
            win.step(*b)
            ref.step(*b)
        assert win._pending
        got = read(win)
        assert not win._pending, name
        want = read(ref)
        if name == "stats":     # fp32 sums in another order
            assert got[1] == want[1] and torch.allclose(got[0], want[0], rtol=1e-5)
        else:
            assert torch.equal(got, want), name
        win.close(); ref.close()
    # close drains too
    win, _ = _pair()
    win.step(*_conflict_free_steps(g, dev, 1, 1, 500, packed=True)[0][0])
    win.close()
    assert not win._pending
    # a non-finite update inside a window
    win, _ = _pair()
    b = _batch(g, dev, 500, USERS, ITEMS, packed=False)
    r = b[2].clone(); r[17] = float("inf")
    win.step(b[0], b[1], r)
    assert win._pending
    with pytest.raises(FactorIsNotANumberException):
        win.check_finite()
    # save -> load round trip of a windowed model
    win, ref = _pair()
    for b in _conflict_free_steps(g, dev, 1, 3, 500, packed=True)[0]:
        win.step(*b)
        ref.step(*b)
    win.save(str(tmp_path / "w"))
    ref.save(str(tmp_path / "r"))
    other, _ = _pair()
    other.load(str(tmp_path / "w"))
    _same_tables(other, ref)


def test_fit_stream_applies_the_window_first_and_reports_each_micro_batch(dev):
    """fit_stream reads the loss of every micro-batch, so it runs per launch: a window pending when it starts
    is applied before its first micro-batch, and windowed steps after it see its updates."""
    win, ref = _pair()
    g = torch.Generator().manual_seed(9)
    before, after = _conflict_free_steps(g, dev, 2, 3, 700, packed=True)
    for b in before:
        win.step(*b)
        ref.step(*b)
    assert len(win._pending) == 3
    host = []
    for step in _conflict_free_steps(g, dev, 5, 5, 700, packed=True):
        host += [tuple(t.cpu().pin_memory() for t in b) for b in step]
    a = list(win.fit_stream(iter(host)))
    b = list(ref.fit_stream(iter(host)))
    for bt in after:
        win.step(*bt)
        ref.step(*bt)
    assert len(a) == len(b) == 25
    for (sa, na), (sb, nb) in zip(a, b):
        assert na == nb == 700
        assert sa == pytest.approx(sb, rel=1e-5)
    _same_tables(win, ref)


def test_graph_step_on_a_windowed_model_matches_eager(dev):
    win, ref = _pair()
    g = torch.Generator().manual_seed(10)
    steps = _conflict_free_steps(g, dev, 3, 3, 600, packed=True)
    win.step(*steps[0][0])         # pending when the graph is made
    ref.step(*steps[0][0])
    static, replay = win.make_graph_step(600, packed=True)
    ref_static, ref_replay = ref.make_graph_step(600, packed=True)
    for step in steps[1:]:
        for b in step:
            static[0].copy_(b[0]); replay()
            ref_static[0].copy_(b[0]); ref_replay()
    win.step(*steps[0][1])         # eager windowed step after replays
    ref.step(*steps[0][1])
    # the graph warm-up steps are all-zero records (one user and one item 600 times): racy in both models
    torch.testing.assert_close(win.users, ref.users, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(win.items.local, ref.items.local, rtol=1e-5, atol=1e-4)


def test_windowed_step_launches_nothing_and_a_drain_is_one_launch(dev):
    from fps_b200.ops import native

    win, _ = _pair()
    g = torch.Generator().manual_seed(12)
    before = native.launch_count()
    for b in _conflict_free_steps(g, dev, 1, 5, 500, packed=False)[0]:
        win.step(*b)
    assert native.launch_count() == before
    win.flush()
    assert native.launch_count() == before + 1
    assert win.stats[1].item() == 2_500


def test_auto_window_follows_the_table_size(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    assert DeviceOnlineMF(1_000, 2_048, 64, seed=1).step_window == 0            # 512 KB item table: off
    big = DeviceOnlineMF(1_000, 300_000, 64, seed=1)                            # 77 MB: on
    assert big.step_window == 8
    os.environ["FPS_STEP_WINDOW"] = "0"
    try:
        assert DeviceOnlineMF(1_000, 300_000, 64, seed=1).step_window == 0
    finally:
        del os.environ["FPS_STEP_WINDOW"]
