"""The one-launch (cooperative) bucket deal of the L2-blocked MF step, and when the step uses it."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _model(blocking, lr=0.05):
    from fps_b200.models.mf.device import DeviceOnlineMF

    return DeviceOnlineMF(30_000, 2_000, 64, learning_rate=lr, seed=5, err_mode=1, item_blocking=blocking,
                          block_bytes=64 << 10)


def test_deal_runs_only_when_rows_are_revisited(dev):
    from fps_b200.ops import native

    m = _model(True)
    assert m.block_buckets == 8
    g = torch.Generator().manual_seed(1)
    for n, launches in ((1_500, 1), (6_000, 2)):          # 2000 item rows: no deal / deal + fused kernel
        u = torch.randperm(30_000, generator=g)[:n].int().to(dev)
        i = torch.randint(0, 2_000, (n,), generator=g, dtype=torch.int32).to(dev)
        before = native.launch_count()
        m.step(u, i, torch.rand(n, generator=g).to(dev))
        assert native.launch_count() - before == launches
    torch.cuda.synchronize()
    assert m.stats[1].item() == 7_500
    m.close()


def test_graph_step_with_bucket_deal_matches_eager(dev):
    """The cooperative deal kernel inside a captured CUDA graph: same updates as eager blocked steps."""
    from fps_b200.ops import native

    n = 8_192                                              # > 2000 rows: every step deals
    g = torch.Generator().manual_seed(2)
    batches = [native.pack_ratings(torch.randperm(30_000, generator=g)[:n].int(),
                                   torch.randint(0, 2_000, (n,), generator=g, dtype=torch.int32),
                                   torch.rand(n, generator=g).half().float()).to(dev) for _ in range(3)]
    eager, graphed = _model(True, lr=0.0), _model(True, lr=0.0)
    (static,), replay = graphed.make_graph_step(n, packed=True)
    U, V = graphed.users.clone(), graphed.items.local.clone()
    graphed.stats.zero_()
    for b in batches:
        eager.stats.zero_(); eager.step(b)
        static.copy_(b); replay()
        torch.cuda.synchronize()
        assert graphed.stats[1].item() == eager.stats[1].item() == n
        torch.testing.assert_close(graphed.stats[0], eager.stats[0], rtol=1e-5, atol=0)
    assert torch.equal(graphed.users, U) and torch.equal(graphed.items.local, V)   # lr = 0: nothing corrupt
    eager.close(); graphed.close()
