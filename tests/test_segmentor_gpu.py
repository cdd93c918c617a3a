"""Segmentor end to end on the GPU: fit (reference training-loop semantics), checkpoint round trip,
predict -> atom coordinates.  API contract of atomai/models/segmentor.py and
test/models/test_loaders.py:63-87."""
import numpy as np
import pytest
import torch

import golden_utils as gu

pytestmark = pytest.mark.gpu


def _data(n, h, w, seed):
    X = gu.images(seed, n, h, w)
    y = gu.labels(seed + 1, n, h, w, 3)
    return X, y


def test_fit_semantics_and_checkpoint_roundtrip(cuda, tmp_path):
    import atomai_b200 as ab
    from atomai_b200.models import Segmentor, load_model
    ab.set_math("tf32")
    X, y = _data(24, 64, 64, 1)
    Xt, yt = _data(8, 64, 64, 5)
    m = Segmentor("Unet", nb_classes=3)
    m.fit(X, y, Xt, yt, training_cycles=6, batch_size=8, print_loss=2,
          filename=str(tmp_path / "seg"), plot_training_history=False)
    assert len(m.loss_acc["train_loss"]) == 6 and len(m.loss_acc["test_loss"]) == 6
    assert all(np.isfinite(m.loss_acc["train_loss"]))
    assert m.loss_acc["train_loss"][-1] < m.loss_acc["train_loss"][0]
    ck = torch.load(str(tmp_path / "seg_metadict_final.tar"), weights_only=False)
    for k in ("model_type", "model", "nb_classes", "batch_norm", "upsampling", "nb_filters",
              "layers", "weights", "optimizer"):
        assert k in ck
    m2 = load_model(str(tmp_path / "seg_metadict_final.tar"))
    for (k1, v1), (k2, v2) in zip(m.net.state_dict().items(), m2.net.state_dict().items()):
        assert k1 == k2 and torch.equal(v1.cpu(), v2.cpu())
    # same seed => same first losses (determinism of the data pipeline; kernels use atomics, so
    # equality is to fp32 tolerance, not bitwise)
    m3 = Segmentor("Unet", nb_classes=3)
    m3.fit(X, y, Xt, yt, training_cycles=6, batch_size=8, filename=str(tmp_path / "seg3"),
           plot_training_history=False)
    np.testing.assert_allclose(m3.loss_acc["train_loss"][:3], m.loss_acc["train_loss"][:3], rtol=2e-3)


def test_host_resident_data_prefetch_matches_device_resident(cuda, tmp_path):
    """Data sets larger than `memory_alloc` stay in (pinned) host memory, as in the reference
    (atomai/utils/preproc.py:170-201); the trainer copies cycle e+1 on a side stream while cycle e
    computes.  Same seed => same losses as the device-resident run."""
    import atomai_b200 as ab
    from atomai_b200.models import Segmentor
    ab.set_math("fp32")
    X, y = _data(32, 32, 32, 11)
    Xt, yt = _data(16, 32, 32, 12)
    losses = []
    for alloc in (4, 0):
        m = Segmentor("Unet", nb_classes=3, nb_filters=8)
        m.fit(X, y, Xt, yt, training_cycles=5, batch_size=8, memory_alloc=alloc,
              filename=str(tmp_path / f"pf{alloc}"), plot_training_history=False)
        assert m.X_train[0].is_cuda == (alloc == 4)
        if alloc == 0:
            assert m.X_train[0].is_pinned()
        losses.append((list(m.loss_acc["train_loss"]), list(m.loss_acc["test_loss"])))
    # Two runs of the same code are not bit-identical: the weight-gradient kernels flush their
    # partial sums with fp32 atomics (order varies run to run, ~1e-7), and Adam's first steps turn
    # a 1e-7 difference of a near-zero gradient into a full-size update (measured 4e-5 on the loss
    # after 4 cycles).  A wrong or stale prefetched batch would move the loss by > 1e-2.
    np.testing.assert_allclose(losses[0][0], losses[1][0], rtol=1e-3)
    np.testing.assert_allclose(losses[0][1], losses[1][1], rtol=1e-3)


def test_full_epoch_mode_and_binary_loss(cuda, tmp_path):
    import atomai_b200 as ab
    from atomai_b200.models import Segmentor
    ab.set_math("tf32")
    X = gu.images(3, 16, 32, 32)
    y = (gu.labels(4, 16, 32, 32, 2) > 0).astype(np.int64)
    m = Segmentor("Unet", nb_classes=1, nb_filters=8)
    m.fit(X, y, X[:8], y[:8], training_cycles=2, batch_size=4, full_epoch=True,
          filename=str(tmp_path / "bin"), plot_training_history=False)
    assert str(m.criterion) == "BCEWithLogitsLoss()"
    assert len(m.loss_acc["train_loss"]) == 2


def test_predict_coordinates_match_reference_pipeline(cuda):
    """pretrained bfo weights on the reference's test-image crop: coordinates from the native
    forward (fp32 math) equal those the reference's Locator extracts from the reference's logits."""
    import atomai_b200 as ab
    from atomai_b200.models import Segmentor
    from atomai_b200.predictors import Locator
    ab.set_math("fp32")
    w = gu.load("bfo_weights.npz")
    g = gu.load("bfo_crop.npz")
    m = Segmentor("Unet", nb_classes=3)
    m.net.load_state_dict({k: torch.from_numpy(w[k]) for k in w.files})
    nn_out, coords = m.predict(g["image"], verbose=False)
    assert nn_out.shape == (1, 128, 128, 3) and nn_out.dtype == np.float32
    ref_prob = torch.softmax(torch.from_numpy(g["logits"]), 1).permute(0, 2, 3, 1).numpy()
    ref_coords = Locator(0.5).run(ref_prob)[0]
    assert coords[0].shape == ref_coords.shape
    assert np.abs(coords[0] - ref_coords).max() < 1e-3
    assert np.abs(nn_out - ref_prob).max() < 1e-4


def test_training_is_bitwise_reproducible(cuda, tmp_path):
    """Two fits from the same seed in the default math mode end in bit-identical weights and
    losses: every cross-CTA reduction of the training path (BatchNorm statistics and backward
    sums, weight gradients, the loss) adds its partials in a fixed order.  Adam turns last-bit
    differences of near-zero gradients into full learning-rate steps, so anything less than
    bitwise equality would show up as visibly different weights."""
    import atomai_b200 as ab
    from atomai_b200.models import Segmentor
    ab.set_math("tf32x3")
    X, y = _data(16, 128, 128, 21)
    Xt, yt = _data(8, 128, 128, 23)
    runs = []
    for i in range(2):
        m = Segmentor("Unet", nb_classes=3, seed=1)
        m.fit(X, y, Xt, yt, training_cycles=5, batch_size=8, filename=str(tmp_path / f"r{i}"),
              plot_training_history=False)
        runs.append(({k: v.detach().cpu().clone() for k, v in m.net.state_dict().items()},
                     [float(v) for v in m.loss_acc["train_loss"] + m.loss_acc["test_loss"]]))
    (sd0, l0), (sd1, l1) = runs
    assert l0 == l1
    for k in sd0:
        assert torch.equal(sd0[k], sd1[k]), k
