"""CPU checks of the occupancy-loss oracles and of the module's host logic: the fp64 oracle's analytic gradient against
autograd through the fp64 restatement (stable sort), on small cases and the edge cases the contract names."""
import numpy as np
import pytest
import torch

import occ_loss_oracle as olo
from gaussianformer_b200.loss import OccupancyLoss, occupancy_loss
from gaussianformer_b200.synthetic import make_occ_labels, make_occ_loss_inputs

C = 18
MANUAL = [1.01552756, 1.06897009, 1.30013094, 1.07253735, 0.94637502, 1.10087012, 1.26960524, 1.06258364, 1.189019,
          1.06217292, 1.00595144, 0.85706115, 1.03923299, 0.90867526, 0.8936431, 0.85486129, 0.8527829, 0.5]


def _weights(n=C):
    return np.asarray(MANUAL[:n], np.float64) * n / np.sum(np.abs(MANUAL[:n]))


def _compare(pred, labels, mask, *, use_softmax, lovasz_ignore=17, empty_label=None, ce_weight=10.0,
             lovasz_weight=1.0):
    """oracle value and gradient == fp64 restatement with stable sort, value and autograd gradient"""
    w = _weights(pred.shape[1])
    kw = dict(use_softmax=use_softmax, lovasz_ignore=lovasz_ignore, empty_label=empty_label, ce_weight=ce_weight,
              lovasz_weight=lovasz_weight)
    ref = olo.oracle(pred, labels, mask, w, **kw)
    x = torch.tensor(np.asarray(pred, np.float64), requires_grad=True)
    m = None if mask is None else torch.as_tensor(mask)
    loss, ce, lov = olo.restatement(x, torch.as_tensor(labels), m, torch.as_tensor(w), stable=True, **kw)
    np.testing.assert_allclose(ref["lovasz"], float(lov.detach()), rtol=1e-12, atol=1e-14)
    if np.isnan(ref["ce"]):
        assert torch.isnan(ce)
        return ref
    np.testing.assert_allclose(ref["loss"], float(loss.detach()), rtol=1e-12, atol=1e-14)
    loss.backward()
    np.testing.assert_allclose(ref["grad"], x.grad.numpy(), rtol=1e-10, atol=1e-14)
    return ref


def _small(B=2, N=300, use_softmax=True, seed=0, ignore_share=0.05, n_classes=C):
    pred, labels, mask = make_occ_loss_inputs(B, N, n_classes, use_softmax, seed, ignore_share=ignore_share,
                                              duplicate_share=0.0)
    return pred.transpose(1, 2).numpy(), labels.numpy(), mask.numpy()


@pytest.mark.parametrize("use_softmax", [True, False])
@pytest.mark.parametrize("with_mask", [True, False])
@pytest.mark.parametrize("empty", [None, 17])
def test_oracle_gradient_equals_autograd(use_softmax, with_mask, empty):
    pred, labels, mask = _small(use_softmax=use_softmax, seed=1 + use_softmax)
    ref = _compare(pred, labels, mask if with_mask else None, use_softmax=use_softmax, empty_label=empty)
    assert len(ref["present"]) >= 10
    if empty is None:
        assert (labels.reshape(-1)[ref["V"]] == 255).any()   # 255 stays in V as background


def test_probability_branch_clamp_edges():
    pred, labels, mask = _small(use_softmax=False, seed=3)
    B, _, N = pred.shape
    flat = pred.transpose(0, 2, 1).reshape(B * N, C)
    y = labels.reshape(-1)
    rows = np.nonzero((y < C))[0][:6]
    flat[rows[0], y[rows[0]]] = 0.0                      # below the clamp: no CE gradient
    flat[rows[1], y[rows[1]]] = np.float32(1e-6)         # on the bound: gradient passes
    flat[rows[2], y[rows[2]]] = 1.0                      # above: blocked; also an exact zero Lovasz error
    pred = flat.reshape(B, N, C).transpose(0, 2, 1).copy()
    _compare(pred, labels, None, use_softmax=False)


@pytest.mark.parametrize("use_softmax", [True, False])
def test_empty_mask(use_softmax):
    pred, labels, mask = _small(use_softmax=use_softmax)
    ref = _compare(pred, labels, np.zeros_like(mask), use_softmax=use_softmax)
    assert np.isnan(ref["ce"]) and ref["lovasz"] == 0.0 and not ref["grad"].any() and ref["present"] == []


@pytest.mark.parametrize("use_softmax", [True, False])
def test_no_present_class(use_softmax):
    pred, labels, _ = _small(use_softmax=use_softmax)
    labels = np.where(labels % 2 == 0, 17, 255)          # V holds only 255s: background of every class
    ref = _compare(pred, labels, None, use_softmax=use_softmax)
    assert ref["present"] == [] and ref["lovasz"] == 0.0 and len(ref["V"]) > 0


@pytest.mark.parametrize("use_softmax", [True, False])
def test_single_voxel_in_v(use_softmax):
    pred, labels, _ = _small(use_softmax=use_softmax)
    labels = np.full_like(labels, 17)
    labels[1, 7] = 4
    ref = _compare(pred, labels, None, use_softmax=use_softmax)
    assert len(ref["V"]) == 1 and ref["present"] == [4]


@pytest.mark.parametrize("use_softmax", [True, False])
def test_all_errors_equal(use_softmax):
    B, N = 1, 64
    pred = np.zeros((B, C, N)) if use_softmax else np.full((B, C, N), 0.25)
    labels = np.full((B, N), 3)
    labels[0, ::3] = 5
    ref = _compare(pred, labels, None, use_softmax=use_softmax)
    for c in ref["present"]:   # ties keep ascending position
        e = ref["errors"][c]
        for val in np.unique(e):
            pos = ref["order"][c][np.isin(ref["order"][c], np.nonzero(e == val)[0])]
            assert (np.diff(pos) > 0).all()


def test_loss_value_does_not_depend_on_tie_order():
    pred = np.zeros((1, C, 40))
    labels = np.full((1, 40), 2)
    labels[0, ::4] = 9
    w = _weights()
    kw = dict(use_softmax=True, lovasz_ignore=17, ce_weight=10.0, lovasz_weight=1.0)
    a = olo.oracle(pred, labels, None, w, **kw)
    # descending error, equal errors in DESCENDING position: every tie group reversed
    rev = {c: np.lexsort((-np.arange(len(e)), -e)) for c, e in a["errors"].items()}
    assert any((rev[c] != a["order"][c]).any() for c in rev)
    b = olo.oracle(pred, labels, None, w, order=rev, **kw)
    assert abs(a["loss"] - b["loss"]) < 1e-12


def test_class_weights_as_the_reference_builds_them():
    m = OccupancyLoss(num_classes=C, balance_cls_weight=True, manual_class_weight=MANUAL, use_sem_geo_scal_loss=False,
                      lovasz_ignore=17)
    w = np.asarray(MANUAL, np.float32)
    np.testing.assert_allclose(m.class_weights.numpy(), C * w / np.abs(w).sum(), rtol=1e-6)
    assert "class_weights" not in m.state_dict()
    plain = OccupancyLoss(num_classes=C, use_sem_geo_scal_loss=False)
    assert torch.equal(plain.class_weights, torch.ones(C))


def test_module_keywords():
    m = OccupancyLoss(weight=2.0, empty_label=17, num_classes=C, use_focal_loss=False, use_dice_loss=False,
                      balance_cls_weight=True, multi_loss_weights=dict(loss_voxel_ce_weight=10.0,
                                                                       loss_voxel_lovasz_weight=1.0),
                      use_sem_geo_scal_loss=False, use_lovasz_loss=True, lovasz_ignore=17,
                      manual_class_weight=MANUAL, lovasz_use_softmax=False,
                      input_dict=dict(pred_occ="p", sampled_xyz="x", sampled_label="l", occ_mask="m"))
    assert (m.weight, m.loss_voxel_ce_weight, m.loss_voxel_lovasz_weight, m.lovasz_ignore) == (2.0, 10.0, 1.0, 17)
    assert m.input_dict["pred_occ"] == "p" and m.loss_func == m.loss_voxel and not m.lovasz_use_softmax
    assert OccupancyLoss(use_sem_geo_scal_loss=False).input_dict == {
        "pred_occ": "pred_occ", "sampled_xyz": "sampled_xyz", "sampled_label": "sampled_label", "occ_mask": "occ_mask"}
    for bad in ("use_focal_loss", "use_dice_loss", "use_sem_geo_scal_loss"):
        kw = dict(use_sem_geo_scal_loss=False)
        kw[bad] = True
        with pytest.raises(NotImplementedError, match=bad):
            OccupancyLoss(**kw)
    with pytest.raises(NotImplementedError, match="manual_class_weight"):
        OccupancyLoss(balance_cls_weight=True, use_sem_geo_scal_loss=False)


def test_op_refuses_cpu_tensors():
    pred, labels, mask = make_occ_loss_inputs(1, 50, C, True, 0)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        occupancy_loss(pred.transpose(1, 2), labels, mask, class_weights=torch.ones(C), ce_weight=10.0,
                       lovasz_weight=1.0, lovasz_ignore=17)


def test_synthetic_labels():
    y = make_occ_labels(2, 200000, C, seed=0, ignore_share=0.01)
    share = lambda v: float((y == v).float().mean())
    assert 0.86 < share(17) < 0.885 and 0.02 < share(0) < 0.04 and 0.005 < share(255) < 0.015
    assert all((y == c).any() for c in range(C))
    pred, labels, mask = make_occ_loss_inputs(1, 1000, C, False, 0, duplicate_share=0.05)
    assert pred.shape == (1, 1000, C) and pred.is_contiguous() and torch.equal(mask, labels != 0)
    assert torch.allclose(pred.sum(-1), torch.ones(1, 1000), atol=1e-5)
