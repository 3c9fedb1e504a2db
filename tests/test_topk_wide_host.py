"""Row-width limit of the device top-K, checked before anything reaches a GPU."""
import pytest
import torch


def test_device_topk_rejects_rows_wider_than_512_on_construction():
    from fps_b200.models.mf.device_topk import DeviceTopK

    with pytest.raises(ValueError, match="at most 512 floats"):
        DeviceTopK(torch.zeros(10, 516))


def test_native_topk_calls_reject_rows_wider_than_512():
    from fps_b200.ops import native

    assert native.TOPK_MAX_STRIDE == 512
    native.check_topk_stride(512)
    items = torch.zeros(10, 516)
    with pytest.raises(ValueError, match="at most 512 floats"):
        native.topk_geometry(items, 4)
    with pytest.raises(ValueError, match="at most 512 floats"):
        native.topk_mma(items, 0, q_local=torch.zeros(4, 516), out_scores=torch.zeros(4, 10))
