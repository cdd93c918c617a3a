"""MSE / BCE-with-logits choose between the operands' own memory order and contiguous copies by
`losses._dense_layout`; pinned here for the layouts the models produce, including prediction and
target with identical strides (the (N, out) Regressor output)."""
import pytest
import torch

from atomai_b200.losses_metrics.losses import _dense_layout


def test_dense_layout():
    assert _dense_layout(torch.zeros(4, 2))
    assert _dense_layout(torch.zeros(4, 1, 5, 5).permute(0, 2, 3, 1))    # channels-last view
    assert _dense_layout(torch.zeros(3, 4, 5).permute(2, 0, 1))
    assert _dense_layout(torch.zeros(1, 1))
    assert not _dense_layout(torch.zeros(4, 6)[:, :3])                     # channel slice
    assert not _dense_layout(torch.zeros(4, 6)[:, ::2])
    assert not _dense_layout(torch.zeros(3, 1).expand(3, 4))               # overlapping


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["same_strides", "sliced", "permuted"])
def test_mse_and_bce_layouts(cuda, layout):
    from atomai_b200.losses_metrics import BCEWithLogitsLoss, MSELoss
    g = torch.Generator().manual_seed(0)
    base_p, base_t = torch.randn(6, 8, generator=g), torch.rand(6, 8, generator=g)
    if layout == "same_strides":
        p, t = base_p[:, :3].contiguous(), base_t[:, :3].contiguous()
    elif layout == "sliced":
        p, t = base_p[:, :3], base_t[:, :3].contiguous()
    else:
        p, t = base_p.t(), base_t.t().contiguous()
    for native, ref in ((MSELoss(), torch.nn.functional.mse_loss),
                        (BCEWithLogitsLoss(), torch.nn.functional.binary_cross_entropy_with_logits)):
        pc = p.to(cuda).requires_grad_(True)
        loss = native(pc, t.to(cuda))
        loss.backward()
        pr = p.double().requires_grad_(True)
        lr = ref(pr, t.double())
        lr.backward()
        assert abs(loss.item() - lr.item()) < 1e-5 * max(1.0, abs(lr.item()))
        assert torch.allclose(pc.grad.cpu().double(), pr.grad, atol=1e-6)
