"""Shared test helpers: seeded inputs -> oracle results (numpy) in the layouts the ops return."""
import numpy as np
import torch

import oracle
from gaussianformer_b200.synthetic import make_splat_inputs

# fp32 parity gate of the splat op (BASELINE.md "Parity gates"): |new - ref| <= ATOL + RTOL * |ref|
RTOL, ATOL = 1e-4, 1e-5


def splat_case(name, seed=0, perturb=False, overrides=None, variant=None, per_axis=False):
    kw, inp, var = make_splat_inputs(name, seed=seed, perturb=perturb, overrides=overrides)
    variant = variant or var
    if per_axis:
        variant = "prob_fast"
    return kw, inp, variant


def oracle_prep(kw, inp, variant):
    a = {k: v[0].numpy() for k, v in inp.items()}
    dims = (kw["H"], kw["W"], kw["D"])
    pi, mi, radii = oracle.host_prep(a["pts"], a["means"], a["scales"], kw["pc_min"], kw["grid_size"],
                                     kw["scale_multiplier"], radii_min=None if variant == "base" else 1,
                                     per_axis=variant == "prob_fast", dims=None)
    return a, pi, mi, radii, oracle.cov6_from_3x3(a["cov"]), dims


def oracle_forward(kw, inp, variant, precision="f64"):
    a, pi, mi, radii, cov6, dims = oracle_prep(kw, inp, variant)
    if variant == "base":
        out, R = oracle.splat_forward(a["pts"], pi, a["means"], mi, a["opa"], a["sem"], cov6, radii, dims, precision)
        return dict(logits=out, num_pairs=R)
    lg, bl, de, pr, R = oracle.splat_prob_forward(a["pts"], pi, a["means"], mi, a["opa"], a["sem"], cov6, radii, dims,
                                                  precision)
    return dict(logits=lg, bin_logits=bl, density=de, probability=pr, num_pairs=R)


def oracle_backward(kw, inp, variant, grads, saved=None, precision="f64"):
    a, pi, mi, radii, cov6, dims = oracle_prep(kw, inp, variant)
    if variant == "base":
        return oracle.splat_backward(a["pts"], pi, a["means"], mi, a["opa"], a["sem"], cov6, radii, dims, grads[0],
                                     precision)
    return oracle.splat_prob_backward(a["pts"], pi, a["means"], mi, a["opa"], a["sem"], cov6, radii, dims,
                                      saved["logits"], saved["bin_logits"], saved["probability"], grads[0], grads[1],
                                      grads[2], precision)


def make_module(kw, variant, device="cuda", validate=True):
    from gaussianformer_b200.splat import LocalAggregator, LocalAggregatorProb, LocalAggregatorProbFast
    cls = {"base": LocalAggregator, "prob": LocalAggregatorProb, "prob_fast": LocalAggregatorProbFast}[variant]
    m = cls(**kw).to(device)
    m.validate = validate
    return m


def to_dev(inp, device="cuda", requires_grad=False):
    t = {k: v.to(device) for k, v in inp.items()}
    if requires_grad:
        for k in ("means", "opa", "sem", "cov"):
            t[k].requires_grad_(True)
    return t


def outside_tolerance(actual, expected, tol):
    """(mask of the entries with |actual - expected| > tol, |actual - expected|, index of the worst one or None).  A NaN
    or an infinity is outside unless both sides hold the same value: ``err > tol`` alone is False for a NaN, so a kernel
    that leaves rows unwritten or sums uninitialised memory would pass."""
    with np.errstate(invalid="ignore"):   # inf - inf
        err = np.abs(actual - expected)
        bad = ~((err <= tol) | (actual == expected) | (np.isnan(actual) & np.isnan(expected)))
    if not bad.any():
        return bad, err, None
    return bad, err, np.unravel_index(np.argmax(np.where(bad, np.nan_to_num(err - tol, nan=np.inf), -np.inf)), err.shape)


def assert_close(actual, expected, rtol=RTOL, atol=ATOL, what=""):
    actual = np.asarray(actual, dtype=np.float64)
    expected = np.asarray(expected, dtype=np.float64)
    tol = atol + rtol * np.abs(expected)
    bad, err, i = outside_tolerance(actual, expected, tol)
    if bad.any():
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.size} outside tolerance; worst at {i}: "
                             f"got {actual[i]!r} want {expected[i]!r} (|err|={err[i]:.3e}, tol={tol[i]:.3e})")


def grad_tolerance(ref):
    """Absolute slack for comparing two DIFFERENT fp32 evaluations of the same gradient with each other (e.g. a
    batched against a per-sample launch, whose atomics add in another order): 2e-4 of the tensor's own scale.
    Parity against the oracle / the reference op does not use this -- see assert_grad_parity."""
    ref = np.asarray(ref, np.float64)
    return 2e-4 * max(1.0, float(np.abs(ref).max()))


K_FLOOR = 4.0


def assert_grad_parity(mine, ref64, ref32, what="", k=K_FLOOR, extra_floor=0.0):
    """Gradient parity gate.  BASELINE.md states ``|new - ref| <= 1e-5 + 1e-4*|ref|`` for gradients too; an entry
    is a sum of 10^2..10^6 signed fp32 terms, so where that cannot hold the bound is the MEASURED fp32 floor of the
    reference arithmetic on the same tensor: ``k * max|fp32 oracle - fp64 oracle|`` (``extra_floor``: the same
    figure for a reference-op golden, when one is compared).  Measured at the BASELINE sizes: cfg 2 and 3 hold the
    elementwise gate on every entry; the prob configs leave <= 60 of 10^5 entries to the floor rule, with the new op
    1-20x CLOSER to the fp64 oracle than the reference op."""
    mine = np.asarray(mine, np.float64)
    ref64 = np.asarray(ref64, np.float64)
    floor = max(float(np.abs(np.asarray(ref32, np.float64) - ref64).max()), float(extra_floor))
    tol = np.maximum(ATOL + RTOL * np.abs(ref64), k * floor)
    bad, err, i = outside_tolerance(mine, ref64, tol)
    if bad.any():
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.size} outside max(1e-5 + 1e-4|ref|, {k} x fp32 floor {floor:.3e}); "
                             f"worst at {i}: got {mine[i]!r} want {ref64[i]!r} (|err|={err[i]:.3e})")


def oracle_grads(kw, inp, variant, grads, saved_from=None):
    """(fp64, fp32) oracle gradients as dicts means / opa / sem / cov([G,3,3]).  ``saved_from``: for the prob variants
    the forward outputs the backward receives (dict logits / bin_logits / probability); default = the oracle's own
    forward at the same precision."""
    out = []
    for precision in ("f64", "f32"):
        saved = None
        if variant != "base":
            saved = saved_from if saved_from is not None else oracle_forward(kw, inp, variant, precision)
        gm, go, gs, gc = oracle_backward(kw, inp, variant, grads, saved, precision)
        out.append({"means": gm, "opa": go, "sem": gs, "cov": oracle.cov6_grad_to_3x3(gc)})
    return out


def check_module_grads(t, kw, inp, variant, grads, what="", saved_from=None, golden=None, sample=0):
    """Gradients accumulated on the leaf tensors ``t`` (batch entry ``sample``; ``inp`` holds that sample alone)
    against the oracle with assert_grad_parity.
    ``golden``: optional dict of reference-op gradients (same keys): the new op is also compared with it, the
    slack being the golden's own measured distance from the fp64 oracle."""
    g64, g32 = oracle_grads(kw, inp, variant, grads, saved_from)
    for name in ("means", "opa", "sem", "cov"):
        mine = t[name].grad[sample].detach().cpu().numpy()
        assert_grad_parity(mine, g64[name], g32[name], what=f"{what} grad {name}")
        if golden is not None:
            gold = np.asarray(golden[name], np.float64)
            floor = float(np.abs(gold - np.asarray(g64[name], np.float64)).max())
            err = np.abs(mine.astype(np.float64) - gold)
            tol = np.maximum(ATOL + RTOL * np.abs(gold), (K_FLOOR + 1.0) * max(floor, float(np.abs(np.asarray(g32[name], np.float64) - g64[name]).max())))
            assert (err <= tol).all(), f"{what} grad {name} vs reference-op golden: {int((err > tol).sum())} outside, max err {err.max():.3e}"


def tie_voxels(expected):
    """voxels whose top two classes are within twice the elementwise tolerance of each other (numerical ties)"""
    srt = np.sort(np.asarray(expected, np.float64), axis=1)
    return (srt[:, -1] - srt[:, -2]) <= 2 * (ATOL + RTOL * np.abs(srt[:, -1]))


def assert_argmax_parity(actual, expected, min_agree=0.9999):
    """Occupancy prediction parity: the arg-max class must agree on >= 99.99 % of the voxels whose
    decision is not a numerical tie (top-two margin of the reference above twice the tolerance);
    a flip on a decided voxel is an error."""
    actual = np.asarray(actual, np.float64)
    expected = np.asarray(expected, np.float64)
    am, ae = actual.argmax(1), expected.argmax(1)
    rows = np.arange(expected.shape[0])
    margin = expected[rows, ae] - expected[rows, am]
    tol = 2 * (ATOL + RTOL * np.abs(expected[rows, ae]))
    decided_flip = (am != ae) & (margin > tol)
    assert not decided_flip.any(), f"{int(decided_flip.sum())} arg-max flips on decided voxels"
    srt = np.sort(expected, axis=1)
    decided = (srt[:, -1] - srt[:, -2]) > 2 * (ATOL + RTOL * np.abs(srt[:, -1]))
    if decided.any():
        assert (am == ae)[decided].mean() >= min_agree
