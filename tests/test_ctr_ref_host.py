"""The fp64 replay of the wide-&-deep tower (tests/ctr_ref.py) against torch autograd in float64, its ReLU margin
sampler, and every deliberate break.  CPU only."""
import numpy as np
import pytest
import torch

from tests import ctr_ref

H = ctr_ref.H


def case(seed, F, E, B, stride=None, lr=0.05, zero_example=None, frac_labels=False):
    """fp32 inputs of one launch.  ``zero_example``: that example's embedding inputs are all 0 and ``b1`` has zeros
    in the hidden units ``ZERO_UNITS``, whose pre-activation is then exactly 0 for it."""
    rng = np.random.default_rng(seed)
    stride = E + 1 if stride is None else stride
    rows = np.zeros((B * F, stride), dtype=np.float32)
    rows[:, :E + 1] = rng.normal(0, 0.3, (B * F, E + 1)).astype(np.float32)
    W1 = rng.normal(0, 0.2, (F * E, H)).astype(np.float32)
    fixed = ()
    if zero_example is not None:
        rows[zero_example * F:(zero_example + 1) * F, :E] = 0
        fixed = ZERO_UNITS
        x, _ = ctr_ref.split_rows(rows, F, E)
        for j in fixed:                                   # b1 = 0 there: keep the other examples clear by W1 instead
            for _ in range(4096):
                pre, tpre = ctr_ref.pre_activations(x, W1[:, j:j + 1], np.zeros(1))
                live = np.arange(B) != zero_example
                if (np.abs(pre[live]) > ctr_ref.RELU_MARGIN * tpre[live]).all():
                    break
                W1[:, j] = rng.normal(0, 0.2, F * E).astype(np.float32)
            else:
                raise RuntimeError("no W1 column keeps the batch clear of 0")
    x, _ = ctr_ref.split_rows(rows, F, E)
    b1 = ctr_ref.make_b1(rng, x, W1, fixed_zero=fixed)
    w2 = rng.normal(0, 0.3, H).astype(np.float32)
    b2 = rng.normal(0, 0.1, 1).astype(np.float32)
    labels = (rng.random(B).astype(np.float32) if frac_labels else (rng.random(B) < 0.4).astype(np.float32))
    return dict(rows=rows, labels=labels, F=F, E=E, W1=W1, b1=b1, w2=w2, b2=b2, lr=np.float32(lr))


ZERO_UNITS = (0, 5, 77)


def autograd(c, train=True):
    """The same step written with torch autograd in float64."""
    F, E = c["F"], c["E"]
    B = c["labels"].shape[0]
    t = {k: torch.tensor(np.asarray(c[k], dtype=np.float64), requires_grad=True)
         for k in ("rows", "W1", "b1", "w2", "b2")}
    y = torch.tensor(c["labels"], dtype=torch.float64)
    x = t["rows"][:, :E].reshape(B, F * E)
    logit = torch.relu(x @ t["W1"] + t["b1"]) @ t["w2"] + t["b2"] + t["rows"][:, E].reshape(B, F).sum(1)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(logit, y, reduction="sum")
    out = {"prob": torch.sigmoid(logit).detach().numpy(), "loss_sum": float(loss.detach())}
    if train:
        loss.backward()
        lr = float(c["lr"])
        scale = float(np.float32(np.float32(lr) / np.float32(B)))
        out["d_rows"] = (-lr * t["rows"].grad).numpy()
        for k in ("W1", "b1", "w2", "b2"):
            out[k] = (t[k] - scale * t[k].grad).detach().numpy()
        out["W1T"] = out["W1"].T
    return out


def _close(ref, want, fields):
    for k in fields:
        np.testing.assert_allclose(np.asarray(ref[k]).reshape(np.shape(want[k])), want[k], rtol=1e-10, atol=1e-13,
                                   err_msg=k)


SHAPES = [(1, 1, 1), (7, 1, 33), (1, 31, 32), (4, 8, 31), (3, 11, 65), (26, 8, 40), (16, 16, 20)]


@pytest.mark.parametrize("F,E,B", SHAPES)
@pytest.mark.parametrize("train", [True, False])
def test_replay_matches_float64_autograd(F, E, B, train):
    c = case(10 * F + E, F, E, B, stride=E + 4, frac_labels=B % 2 == 1)
    ref = ctr_ref.replay(**c, train=train)
    want = autograd(c, train)
    _close(ref, want, ("prob", "loss_sum") + (("d_rows", "W1", "W1T", "b1", "w2", "b2") if train else ()))
    assert ref["count"] == B
    if train:
        assert (ref["d_rows"][:, E + 1:] == 0).all() and (ref["tol_d_rows"][:, E + 1:] == 0).all()
    else:
        assert "d_rows" not in ref


def test_relu_at_zero_has_zero_gradient():
    c = case(5, 4, 8, 33, zero_example=7)
    ref = ctr_ref.replay(**c)
    assert (ref["pre"][7, list(ZERO_UNITS)] == 0).all()
    _close(ref, autograd(c), ("d_rows", "W1", "b1", "w2", "b2"))   # torch's relu'(0) is 0 as well
    zero = np.zeros_like(ref["pre"], dtype=bool)
    zero[7, list(ZERO_UNITS)] = True
    assert ctr_ref.relu_margin(ref["pre"], ref["tol_pre"], zero) > ctr_ref.RELU_MARGIN


@pytest.mark.parametrize("F,E,B", [(1, 1, 200), (26, 8, 100), (16, 16, 64)])
def test_b1_sampler_keeps_every_preactivation_clear(F, E, B):
    c = case(F + E + B, F, E, B)
    x, _ = ctr_ref.split_rows(c["rows"], F, E)
    pre, tpre = ctr_ref.pre_activations(x, c["W1"], c["b1"])
    assert (np.abs(pre) > ctr_ref.RELU_MARGIN * tpre).all()
    assert 0 < (pre > 0).mean() < 1                         # the units are not all on or all off


def test_prefix_bound_covers_fp32_fma_chains():
    """The ``pre`` bound holds for a float32 in-order chain (numpy float32 rounds each product and each sum, which the
    chain's FMAs only improve on)."""
    rng = np.random.default_rng(2)
    x = rng.normal(0, 1, (64, 256)).astype(np.float32)
    W1 = rng.normal(0, 1, (256, 8)).astype(np.float32)
    b1 = rng.normal(0, 1, 8).astype(np.float32)
    pre, tpre = ctr_ref.pre_activations(x, W1, b1)
    acc = np.broadcast_to(b1, (64, 8)).astype(np.float32).copy()
    for i in range(256):
        acc = (acc + x[:, i:i + 1] * W1[i][None, :]).astype(np.float32)
    assert (np.abs(acc - pre) <= 2 * tpre).all()


def test_every_break_changes_the_result():
    c = case(9, 4, 8, 33, zero_example=3)                 # B % 32 != 0: one partial tile; lr != 1
    ref = ctr_ref.replay(**c)
    for b in ctr_ref.BREAKS:
        bad = ctr_ref.violations(ctr_ref.replay(**c, breaks=b), ref)
        assert bad, b
    with pytest.raises(ValueError):
        ctr_ref.replay(**c, breaks="nope")


def test_fractional_labels_and_large_logits():
    c = case(4, 2, 3, 50, frac_labels=True)
    c["b2"] = np.array([28.0], dtype=np.float32)        # logits near +-30 through the bias
    for b2 in (28.0, -28.0):
        c["b2"] = np.array([b2], dtype=np.float32)
        ref = ctr_ref.replay(**c)
        _close(ref, autograd(c), ("prob", "loss_sum", "d_rows", "W1", "b1", "w2", "b2"))
        assert np.isfinite(ref["tol_loss_sum"]) and (ref["tol_prob"] > 0).all()
