"""Oracle of the splat op's scales-and-rotations route (``forward_from_srt``), the whole chain in one precision:

* Sigma^-1 = R^T diag(1/s^2) R by ``inverse_covariance_from_srt`` in the chain's dtype, rounded once to fp32 (the C
  oracle reads fp32 Sigma^-1);
* the splat forward and backward of the C oracle at the chain's precision;
* the gradients of the scales and the quaternions by autograd through the closed form in the chain's dtype, seeded with
  the oracle's [G,6] gradient of Sigma^-1 on the six gathered entries of the 3x3 (the lower triangle carries none,
  ``__init__.py:143``).  The radii come from the fixed scales and carry no gradient, as in the reference.

The fp64 chain is the reference; the fp32 chain measures the floor of fp32 arithmetic on the same inputs."""
import numpy as np
import torch

import helpers as h
import oracle

GRADS = ("means", "opa", "sem", "scales", "rotations")
OUTPUTS = ("logits", "bin_logits", "density")
_DTYPE = {"f64": torch.float64, "f32": torch.float32}


def srt_chain(kw, inp, scales, rotations, variant, upstream, precision="f64", op_outputs=None):
    """One sample.  ``inp``: the sample's tensors with their leading batch dimension of 1 (``inp["cov"]`` is ignored);
    ``scales [G,3]``, ``rotations [G,4]``: the fp32 values the op reads; ``upstream``: the numpy upstream gradients of
    the op's outputs.  ``op_outputs``: for the prob variants the op's own forward outputs (logits, bin_logits), which
    its backward receives -- the backward then gets them and the fp32 oracle's probability, as
    ``test_splat_routes_gpu._saved`` does; default: this chain's own forward.

    Returns (outputs, grads): the oracle's forward dict, and numpy gradients ``means opa sem scales rotations`` plus
    ``cov`` (the [G,6] gradient of Sigma^-1, for diagnostics)."""
    from gaussianformer_b200.splat import inverse_covariance_from_srt
    dt = _DTYPE[precision]
    s = scales.detach().cpu().to(dt).requires_grad_(True)
    q = rotations.detach().cpu().to(dt).requires_grad_(True)
    cov = inverse_covariance_from_srt(s, q)
    one = dict(inp, scales=scales.detach().cpu().float()[None], cov=cov.detach().float()[None])
    fw = h.oracle_forward(kw, one, variant, precision)
    saved = None
    if variant != "base":
        saved = dict(logits=fw["logits"], bin_logits=fw["bin_logits"], probability=fw["probability"])
        if op_outputs is not None:
            saved = dict(logits=np.asarray(op_outputs[0], np.float32), bin_logits=np.asarray(op_outputs[1], np.float32),
                         probability=h.oracle_forward(kw, one, variant, "f32")["probability"])
    gm, go, gs, gc = h.oracle_backward(kw, one, variant, upstream, saved, precision)
    seed = torch.from_numpy(np.ascontiguousarray(oracle.cov6_grad_to_3x3(gc))).to(dt)
    g_s, g_q = torch.autograd.grad(cov, (s, q), seed)
    grads = dict(means=gm, opa=go, sem=gs, scales=g_s.numpy(), rotations=g_q.numpy(), cov=np.asarray(gc))
    return fw, grads


def srt_chains(kw, inp, scales, rotations, variant, upstream, op_outputs=None):
    """(fp64 chain, fp32 chain), each as srt_chain returns it"""
    return tuple(srt_chain(kw, inp, scales, rotations, variant, upstream, p, op_outputs) for p in ("f64", "f32"))


# ------------------------------------------------------------------------------------------------ gates
def _elementwise_tol(ref):
    return h.ATOL + h.RTOL * np.abs(ref)


def check_outputs(mine, out64, out32, variant, what):
    """The op's outputs (numpy, in OUTPUTS order) against the fp64 chain: helpers.assert_close, the prob variants without
    the voxels on the probability switch.  An output on which the fp32 chain itself misses the elementwise gate (an
    ill-conditioned Sigma^-1 through the prob determinant) is held to helpers.assert_grad_parity with the fp32 chain's
    floor instead, and the number of entries that took the floor is printed.  Returns {output: worst error as a fraction
    of its elementwise tolerance}."""
    names = ("logits",) if variant == "base" else OUTPUTS
    stable = None if variant == "base" else np.abs(out64["probability"] - 1e-9) > 1e-10
    worst = {}
    for name, a in zip(names, mine):
        a, want, w32 = (np.asarray(x, np.float64) for x in (a, out64[name], out32[name]))
        if name == "logits" and stable is not None:
            a, want, w32 = a[stable], want[stable], w32[stable]
        tol = _elementwise_tol(want)
        err = np.abs(a - want)
        worst[name] = float((err / tol).max())
        fp32_misses = int((np.abs(w32 - want) > tol).sum())
        if fp32_misses:
            h.assert_grad_parity(a, want, w32, what=f"{what} {name}")
            print(f"{what} {name}: the fp32 chain misses the elementwise gate on {fp32_misses} entries; "
                  f"{int((err > tol).sum())} of {err.size} entries of the op took the fp32 floor")
        else:
            h.assert_close(a, want, what=f"{what} {name}")
    return worst


def zero_pass_fraction(ref64, ref32, k=h.K_FLOOR):
    """share of the entries an all-zero answer would pass under helpers.assert_grad_parity"""
    ref64 = np.asarray(ref64, np.float64)
    floor = float(np.abs(np.asarray(ref32, np.float64) - ref64).max())
    return float((np.abs(ref64) <= np.maximum(_elementwise_tol(ref64), k * floor)).mean())


def check_grads(mine, g64, g32, what):
    """The op's five gradients (dict of numpy arrays) against the fp64 chain with helpers.assert_grad_parity.  Returns
    (entries outside the elementwise gate per gradient, i.e. the ones that took the floor rule; the share of the
    dL/dscales entries an all-zero answer would pass)."""
    floored = {}
    for name in GRADS:
        a, want = np.asarray(mine[name], np.float64), np.asarray(g64[name], np.float64)
        h.assert_grad_parity(a, want, g32[name], what=f"{what} grad {name}")
        floored[name] = int((np.abs(a - want) > _elementwise_tol(want)).sum())
    return floored, zero_pass_fraction(g64["scales"], g32["scales"])


def check_sample(mine_out, mine_grads, chains, variant, what):
    """outputs and gradients of one sample against (fp64 chain, fp32 chain); prints one report line"""
    (out64, g64), (out32, g32) = chains
    worst = check_outputs(mine_out, out64, out32, variant, what)
    floored, zero = check_grads(mine_grads, g64, g32, what)
    print(f"[srt] {what}: worst output error / tolerance {', '.join(f'{k} {v:.3f}' for k, v in worst.items())}; "
          f"gradient entries on the floor rule {floored}; all-zero dL/dscales would pass {100 * zero:.2f} %")
    return dict(worst=worst, floored=floored, zero_pass=zero)
