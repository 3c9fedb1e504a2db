"""The fused wide-&-deep tower (ops/csrc/fps_ctr.cu) launch by launch against the fp64 replay of tests/ctr_ref.py.

Every case reads the state, runs one ``native.ctr_step``, reads the state back and compares every element within
``MARGIN`` times the replay's bound.  The batches reach every input width the kernel stages (IN = F E from 1 to 256,
with E = 1 and F = 1), row strides with and without padding columns, one example, partial last tiles and grids whose
CTAs walk two and three tiles each; forward-only launches; three consecutive steps; and the whole
``DeviceWideAndDeep.step`` (credit-limited gather, tower, push of duplicate slots)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import ctr_ref
from tests.test_ctr_ref_host import ZERO_UNITS, case

pytestmark = pytest.mark.gpu

MARGIN = ctr_ref.MARGIN
SENTINEL = 1234.5
# (F, E) for IN = 1, 7, 31, 32, 33, 208, 255, 256
PAIRS = [(1, 1), (7, 1), (1, 31), (4, 8), (3, 11), (26, 8), (5, 51), (16, 16)]


def _sm():
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    return native.sm_count(0)


def _padded(E):
    return (E + 1 + 3) // 4 * 4 + 4


def _launch(c, train=True, d_rows="sentinel", grads_fill=0.0, prob=True):
    """One ``native.ctr_step`` on the case's state; every output and the state after, as numpy."""
    from fps_b200.ops import native

    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)   # noqa: E731
    rows, labels = t(c["rows"]), t(c["labels"])
    W1 = t(c["W1"])
    w = {"W1": W1, "W1T": W1.t().contiguous(), "b1": t(c["b1"]), "w2": t(c["w2"]), "b2": t(c["b2"])}
    g = {k: torch.full_like(v, grads_fill) for k, v in w.items() if k != "W1T"}
    dr = torch.full_like(rows, SENTINEL) if d_rows == "sentinel" else None
    loss = torch.zeros(2, device=dev)
    p = torch.full((labels.numel(),), SENTINEL, device=dev) if prob else None
    before = {k: v.clone() for k, v in w.items()}
    native.ctr_step(rows, labels, c["F"], c["E"], w, g, dr, loss, float(c["lr"]), train=train, prob=p)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in w.items()}
    out.update(loss_sum=float(loss[0]), count=float(loss[1]), before={k: v.cpu().numpy() for k, v in before.items()},
               grads={k: v.cpu().numpy() for k, v in g.items()})
    if dr is not None:
        out["d_rows"] = dr.cpu().numpy()
    if p is not None:
        out["prob"] = p.cpu().numpy()
    return out


def _check(c, got, train=True, zero=None):
    """Compare one launch with the replay; returns the replay."""
    ref = ctr_ref.replay(**c, train=train)
    B, E = c["labels"].shape[0], c["E"]
    assert ctr_ref.relu_margin(ref["pre"], ref["tol_pre"], zero) > MARGIN, "a pre-activation is too close to 0"
    assert got["count"] == B
    fields = ctr_ref.FIELDS if train else ("prob", "loss_sum")
    bad = ctr_ref.violations(ref, got, fields)
    assert not bad, bad
    if train:
        assert not (got["d_rows"] == SENTINEL).any()
        assert (got["d_rows"][:, E + 1:] == 0).all()
        assert np.array_equal(got["W1T"], got["W1"].T)
        for k, v in got["grads"].items():
            assert (v == 0).all(), k
    else:
        for k in got["before"]:
            assert np.array_equal(got[k], got["before"][k]), k
    return ref


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("F,E", PAIRS)
def test_input_widths_and_strides(F, E, padded):
    _sm()
    stride = _padded(E) if padded else E + 1
    c = case(100 * F + E + padded, F, E, 777, stride=stride, frac_labels=padded)
    _check(c, _launch(c))


def _batch_sizes(sm):
    return [1, 31, 32, 33, 777, 2 * sm * 32 + 5, 3 * sm * 32]


def test_sweep_reaches_every_width_and_tile_walk():
    """The sweep covers every input width above (with E = 1 and F = 1), and, with the grid min(tiles, SMs), batches
    whose every CTA walks at least two tiles, one of them ending in a partial tile."""
    assert sorted(F * E for F, E in PAIRS) == [1, 7, 31, 32, 33, 208, 255, 256]
    assert any(E == 1 for _, E in PAIRS) and any(F == 1 for F, _ in PAIRS)
    sm = _sm()
    sizes = _batch_sizes(sm)
    least_walk = [ctr_ref.n_tiles(B) // min(ctr_ref.n_tiles(B), sm) for B in sizes]   # tiles every CTA walks
    assert least_walk[:5] == [1] * 5 and least_walk[5] == 2 and least_walk[6] == 3
    assert ctr_ref.padding_examples(sizes[5]) > 0 and ctr_ref.padding_examples(sizes[6]) == 0
    assert [B % 32 for B in sizes[:4]] == [1, 31, 0, 1]


@pytest.mark.parametrize("i", range(7))
@pytest.mark.parametrize("F,E", [(4, 8), (7, 1)])
def test_batch_sizes(F, E, i):
    B = _batch_sizes(_sm())[i]
    c = case(7 * i + F, F, E, B, stride=_padded(E) if i % 2 else E + 1, frac_labels=i % 3 == 0)
    _check(c, _launch(c))


@pytest.mark.parametrize("B_index", [0, 3, 6])
@pytest.mark.parametrize("F,E", [(4, 8), (26, 8), (16, 16)])
def test_forward_only_writes_prob_and_loss_only(F, E, B_index):
    B = _batch_sizes(_sm())[B_index]
    if F * E > 32 and B > 1000:
        B = 777
    c = case(31 * B_index + F, F, E, B, stride=_padded(E), frac_labels=True)
    got = _launch(c, train=False, grads_fill=0.25)
    _check(c, got, train=False)
    assert (got["d_rows"] == SENTINEL).all()
    for k, v in got["grads"].items():
        assert (v == 0.25).all(), k
    got = _launch(c, train=False, d_rows=None)
    _check(c, got, train=False)


def test_relu_at_zero_pins_zero_gradient():
    c = case(5, 4, 8, 33, zero_example=7)
    zero = np.zeros((33, ctr_ref.H), dtype=bool)
    zero[7, list(ZERO_UNITS)] = True
    ref = _check(c, _launch(c), zero=zero)
    assert (ref["pre"][7, list(ZERO_UNITS)] == 0).all()


def test_three_consecutive_steps():
    """Each step is replayed from the kernel's own state before it, so error does not compound.  The learning rate
    is small enough that three steps cannot move a pre-activation across the margin ``make_b1`` left around 0."""
    from fps_b200.ops import native

    sm = _sm()
    dev = torch.device("cuda", 0)
    for F, E, B in [(26, 8, 777), (4, 8, 2 * sm * 32 + 5)]:
        c = case(B + F, F, E, B, stride=_padded(E), lr=1e-5)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)   # noqa: E731
        rows, labels = t(c["rows"]), t(c["labels"])
        W1 = t(c["W1"])
        w = {"W1": W1, "W1T": W1.t().contiguous(), "b1": t(c["b1"]), "w2": t(c["w2"]), "b2": t(c["b2"])}
        g = {k: torch.zeros_like(v) for k, v in w.items() if k != "W1T"}
        for step in range(3):
            state = {k: w[k].cpu().numpy() for k in ("W1", "b1", "w2", "b2")}
            dr = torch.full_like(rows, SENTINEL)
            loss = torch.zeros(2, device=dev)
            prob = torch.empty(B, device=dev)
            native.ctr_step(rows, labels, F, E, w, g, dr, loss, float(c["lr"]), train=True, prob=prob)
            torch.cuda.synchronize()
            got = {k: v.cpu().numpy() for k, v in w.items()}
            got.update(d_rows=dr.cpu().numpy(), prob=prob.cpu().numpy(), loss_sum=float(loss[0]),
                       count=float(loss[1]), grads={k: v.cpu().numpy() for k, v in g.items()})
            _check(dict(c, **state), got)
            assert not np.array_equal(got["W1"], state["W1"]) and not np.array_equal(got["b1"], state["b1"])


def _model_case(pull_limit, seed=3):
    from fps_b200.models.ctr import DeviceWideAndDeep

    _sm()
    dev = torch.device("cuda", 0)
    F, E, B, slots = 6, 8, 777, 4000
    m = DeviceWideAndDeep(slots, F, emb_dim=E, learning_rate=0.05, pull_limit=pull_limit, seed=seed)
    rng = np.random.default_rng(seed)
    hot = rng.integers(0, 40, (B, F))                          # repeated slots across examples
    zipf = np.minimum(rng.zipf(1.3, (B, F)), slots - 1)
    ids = np.where(rng.random((B, F)) < 0.5, hot, zipf).astype(np.int64)
    labels = (rng.random(B) < 0.4).astype(np.float32)
    return m, dev, F, E, B, ids, labels, rng


@pytest.mark.timeout(120)
@pytest.mark.parametrize("pull_limit", [0, 1, 64])
def test_device_wide_and_deep_step_end_to_end(pull_limit):
    m, dev, F, E, B, ids, labels, rng = _model_case(pull_limit)
    table0 = m.table.local.cpu().numpy().astype(np.float64)
    rows = table0[ids.reshape(-1)].astype(np.float32)
    x, _ = ctr_ref.split_rows(rows, F, E)
    m.w["b1"].copy_(torch.from_numpy(ctr_ref.make_b1(rng, x, m.w["W1"].cpu().numpy())))
    state = {k: m.w[k].cpu().numpy() for k in ("W1", "b1", "w2", "b2")}
    ids_d = torch.from_numpy(ids).to(dev)
    loss = m.step(ids_d, torch.from_numpy(labels).to(dev))
    torch.cuda.synchronize()
    assert np.array_equal(m._rows.cpu().numpy(), rows)        # the gather is exact, limiter or not
    c = dict(rows=rows, labels=labels, F=F, E=E, lr=np.float32(m.lr), **state)
    got = {k: v.cpu().numpy() for k, v in m.w.items()}
    got.update(loss_sum=float(loss[0]), count=float(loss[1]), d_rows=m._drows.cpu().numpy(),
               grads={k: v.cpu().numpy() for k, v in m.g.items()})
    ref = _check(c, got)
    # the push: every slot gets the sum of its examples' row gradients, in any order
    flat = ids.reshape(-1)
    want = table0.copy()
    np.add.at(want, flat, ref["d_rows"])
    mag = np.abs(table0).copy()
    np.add.at(mag, flat, np.abs(ref["d_rows"]))
    tol = np.zeros_like(table0)
    np.add.at(tol, flat, ref["tol_d_rows"])
    cnt = np.bincount(flat, minlength=table0.shape[0])[:, None] + 1
    tol += cnt * ctr_ref.EPS * mag
    table1 = m.table.local.cpu().numpy().astype(np.float64)
    bad = ~(np.abs(table1 - want) <= MARGIN * tol)
    assert not bad.any(), np.argwhere(bad)[:5]
    untouched = np.setdiff1d(np.arange(table0.shape[0]), flat)
    assert np.array_equal(table1[untouched], table0[untouched])
    if pull_limit > 0:
        assert int(m.table._credits(pull_limit, dev)[0]) == pull_limit
    # predict through the updated table and weights
    prob = m.predict(ids_d).cpu().numpy()
    after = {k: m.w[k].cpu().numpy() for k in ("W1", "b1", "w2", "b2")}
    rows1 = table1[flat].astype(np.float32)
    fwd = ctr_ref.replay(rows1, labels, F, E, lr=m.lr, train=False, **after)
    assert ctr_ref.relu_margin(fwd["pre"], fwd["tol_pre"]) > MARGIN
    assert not ctr_ref.violations(fwd, {"prob": prob}, ("prob",))
    if pull_limit > 0:
        assert int(m.table._credits(pull_limit, dev)[0]) == pull_limit
    m.close()


def _sensitivity_cases():
    yield case(5, 4, 8, 33, zero_example=7), 7
    for i, (F, E) in enumerate([(1, 1), (7, 1), (4, 8), (26, 8), (16, 16)]):
        yield case(900 + i, F, E, 777 if i % 2 else 95, stride=_padded(E), frac_labels=i % 2 == 0), None


def test_broken_replays_fail():
    _sm()
    counts = {b: 0 for b in ctr_ref.BREAKS}
    cases = 0
    for c, _ in _sensitivity_cases():
        got = _launch(c)
        ref = ctr_ref.replay(**c)
        assert not ctr_ref.violations(ref, got)
        for b in ctr_ref.BREAKS:
            counts[b] += bool(ctr_ref.violations(ctr_ref.replay(**c, breaks=b), got))
        cases += 1
    print(f"\nCTR_SENSITIVITY failing cases of {cases}: {counts}")
    assert all(v > 0 for v in counts.values()), counts


# ---- host refusals: nothing reaches the device ------------------------------------------------------------------
def _valid_args(dev, F=4, E=8, B=40, stride=12):
    IN = F * E
    rows = torch.zeros(B * F, stride, device=dev)
    w = {"W1": torch.zeros(IN, 256, device=dev), "W1T": torch.zeros(256, IN, device=dev),
         "b1": torch.zeros(256, device=dev), "w2": torch.zeros(256, device=dev), "b2": torch.zeros(1, device=dev)}
    g = {k: torch.zeros_like(v) for k, v in w.items() if k != "W1T"}
    return dict(rows=rows, labels=torch.zeros(B, device=dev), fields=F, emb=E, weights=w, grads=g,
                d_rows=torch.zeros_like(rows), loss=torch.zeros(2, device=dev), lr=0.1, train=True,
                prob=torch.zeros(B, device=dev))


def _bad_variants(dev):
    a = _valid_args
    yield "stride == emb", dict(a(dev, stride=8), d_rows=torch.zeros(160, 8, device=dev))
    yield "stride < emb", dict(a(dev, stride=4), d_rows=torch.zeros(160, 4, device=dev))
    yield "rows count", dict(a(dev), rows=torch.zeros(159, 12, device=dev))
    yield "IN > 256", a(dev, F=16, E=17, stride=20)
    for k, shp in [("W1", (33, 256)), ("W1", (256, 32)), ("W1T", (32, 256)), ("b1", (255,)), ("w2", (257,)),
                   ("b2", (2,))]:
        v = a(dev)
        v["weights"][k] = torch.zeros(shp, device=dev)
        yield f"weights {k} {shp}", v
    for k, shp in [("W1", (32, 255)), ("b1", (1,)), ("w2", (128,)), ("b2", (0,))]:
        v = a(dev)
        v["grads"][k] = torch.zeros(shp, device=dev)
        yield f"grads {k} {shp}", v
    yield "prob length", dict(a(dev), prob=torch.zeros(39, device=dev))
    yield "d_rows shape", dict(a(dev), d_rows=torch.zeros(160, 8, device=dev))
    yield "loss size", dict(a(dev), loss=torch.zeros(1, device=dev))


def test_ctr_step_refuses_bad_shapes_before_launching():
    from fps_b200.ops import native

    _sm()
    dev = torch.device("cuda", 0)
    native.ctr_step(**_valid_args(dev))                         # the valid call launches
    torch.cuda.synchronize()
    n = 0
    for what, args in _bad_variants(dev):
        before = native.launch_count()
        with pytest.raises(ValueError):
            native.ctr_step(**args)
        assert native.launch_count() == before, what
        n += 1
    assert n == 17
    torch.cuda.synchronize()


def test_ctr_library_refuses_a_stride_without_the_wide_column():
    """``fps_ctr_step`` itself returns its own code for ``stride < emb + 1``.  The buffers are sized with a spare row
    so that even an unchecked launch would stay inside them."""
    from fps_b200.ops import native

    _sm()
    dev = torch.device("cuda", 0)
    F, E, B = 2, 4, 8
    v = _valid_args(dev, F=F, E=E, B=B, stride=E)
    rows = torch.zeros(B * F + 1, E, device=dev)
    d_rows = torch.zeros(B * F + 1, E, device=dev)
    a = native.CtrArgsC()
    a.rows, a.labels, a.batch, a.fields, a.emb, a.stride = rows.data_ptr(), v["labels"].data_ptr(), B, F, E, E
    for k in ("W1", "W1T", "b1", "w2", "b2"):
        setattr(a, k, v["weights"][k].data_ptr())
    a.gW1, a.gb1, a.gw2, a.gb2 = (v["grads"][k].data_ptr() for k in ("W1", "b1", "w2", "b2"))
    a.d_rows, a.loss, a.prob, a.lr, a.train = d_rows.data_ptr(), v["loss"].data_ptr(), None, 0.1, 1
    w = v["weights"]
    code = native.lib().fps_ctr_step(C.byref(a), *(C.c_void_p(w[k].data_ptr()) for k in ("W1", "W1T", "b1", "w2",
                                                                                            "b2")),
                                     native.sm_count(0), native._stream())
    torch.cuda.synchronize()
    assert code == -1801
    assert b"wide weight" in native.lib().fps_error_string(code)
    assert (d_rows == 0).all() and (v["loss"] == 0).all()
