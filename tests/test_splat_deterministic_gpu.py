"""The splat backward under torch.use_deterministic_algorithms(True): every route (the bin-centric slot route, its
hand-over to the Gaussian-centric chain on a stray point or a slot overflow, and that chain called directly) passes the
fp64-oracle gate and gives identical gradient bytes over repeated calls, a sample alone or inside a batch, and any SM
count.  The inputs of every route are the route matrix of test_splat_routes_gpu.  With the switch off the kernels are
today's.  The deformable-aggregation backwards have no deterministic form and raise / warn through PyTorch's alert."""
import contextlib
import ctypes
import warnings

import pytest
import torch

import helpers as h
import test_parity_full_gpu as full
import test_splat_routes_gpu as routes
from gaussianformer_b200 import _lib

pytestmark = pytest.mark.gpu

CALLS = 3
GRADS = ("means", "opa", "sem", "cov")
NEW_KERNELS = ("slot_plan_kernel", "backward_bin_slots_kernel", "bin_slot_finish_kernel", "queue_scan_kernel",
               "backward_small_det_kernel", "backward_big_det_kernel", "big_finish_kernel")


@contextlib.contextmanager
def deterministic(on=True, warn_only=False):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@contextlib.contextmanager
def plan(slot_budget=-1, num_sms=-1):
    L = _lib.lib()
    L.gf_debug_splat_backward_plan(slot_budget, num_sms)
    try:
        yield
    finally:
        L.gf_debug_splat_backward_plan(-1, -1)


def _bits(x):
    return x.detach().contiguous().view(torch.int32).cpu()


def _grads(kw, inp, variant, offset=0, call=None, seed=7):
    """one forward + backward through the module; the gradients of the leaf tensors as raw bits"""
    m = h.make_module(kw, variant)
    t = h.to_dev(inp, requires_grad=True)
    call = call or (lambda m, t: m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
    outs = routes._outputs(call(m, t))
    _, dev = routes._upstream(outs, seed, offset)
    torch.autograd.backward(list(outs), dev)
    return {k: _bits(t[k].grad) for k in GRADS}


def _assert_same_bits(runs, what):
    for i, r in enumerate(runs[1:], 1):
        for k in r:
            diff = int((r[k] != runs[0][k]).sum())
            assert diff == 0, f"{what}: call {i} differs from call 0 in {diff} entries of grad {k}"


def _repeatable(kw, inp, variant, what, **kw_run):
    runs = [_grads(kw, inp, variant, **kw_run) for _ in range(CALLS)]
    _assert_same_bits(runs, what)
    return runs[0]


# ------------------------------------------------------------------------------------------------ route matrix
def _matrix():
    cases = []
    for variant in routes.VARIANTS:
        for route in routes.ROUTES:
            cases.append((variant, route))
        cases += [(variant, "canonical"), (variant, "mixed_batch"), (variant, "empty_supertile")]
    return cases


def _matrix_inputs(variant, route):
    """(kw, inp, logits-gradient offset, samples that must reach the big-box queue)"""
    if route == "canonical":
        kw, inp = routes._case(variant)
        return kw, inp, 0, ()
    if route == "mixed_batch":
        kw, inp = routes._mixed_batch(variant)
        return kw, inp, 0, (1,)
    if route == "empty_supertile":
        kw, inp = routes._empty_supertile_inputs(variant)
        return kw, inp, 0, None
    kw, inp, offset = routes._route_inputs(variant, route)
    return kw, inp, offset, (0,)


@pytest.mark.parametrize("variant,route", _matrix())
def test_route_matrix_deterministic(variant, route):
    kw, inp, offset, big = _matrix_inputs(variant, route)
    with deterministic():
        routes._check_vs_oracle(kw, inp, variant, f"det {variant}/{route}", offset=offset, big_box=big)
        _repeatable(kw, inp, variant, f"{variant}/{route}", offset=offset)


@pytest.mark.parametrize("variant", routes.VARIANTS)
@pytest.mark.parametrize("order", ["canonical", "permuted"])
def test_forward_from_srt_deterministic(variant, order):
    kw, inp = routes._case(variant)
    G = inp["means"].shape[1]
    gen = torch.Generator().manual_seed(23)
    rots = torch.randn(1, G, 4, generator=gen) * 1.5
    if order == "permuted":
        with deterministic():
            routes.test_forward_from_srt_generic_route(variant)   # the oracle gate of the srt route
        perm = torch.randperm(inp["pts"].shape[1], generator=gen)
        inp = dict(inp, pts=inp["pts"][:, perm].contiguous())
    runs = []
    for _ in range(CALLS):
        m = h.make_module(kw, variant)
        t = h.to_dev(inp)
        leaves = {k: t[k].clone().requires_grad_(True) for k in ("means", "opa", "sem", "scales")}
        leaves["rot"] = rots.cuda().requires_grad_(True)
        with deterministic():
            outs = routes._outputs(m.forward_from_srt(t["pts"], leaves["means"], leaves["opa"], leaves["sem"],
                                                      leaves["scales"], leaves["rot"]))
            torch.autograd.backward(list(outs), routes._upstream(outs, 29)[1])
        runs.append({k: _bits(v.grad) for k, v in leaves.items()})
    _assert_same_bits(runs, f"{variant}/srt {order}")


# ------------------------------------------------------------------------------------------------ full size
@pytest.mark.parametrize("case,cfg,seed,perturb,per_axis", [full.CASES[0], full.CASES[3]], ids=["cfg2", "cfg4_prob"])
def test_full_size_deterministic(case, cfg, seed, perturb, per_axis):
    with deterministic():
        full.test_full_size_vs_reference_op_and_fp64_oracle(case, cfg, seed, perturb, per_axis)
        kw, inp, variant = h.splat_case(cfg, seed, perturb, per_axis=per_axis)
        _repeatable(kw, inp, variant, case)


# ------------------------------------------------------------------------------------------------ batch
def _three(variant, permuted):
    parts = []
    for i in range(3):
        kw, one = routes._case(variant, seed=routes.BASE_INPUTS[variant][1] + 50 + i)
        if permuted:
            perm = torch.randperm(one["pts"].shape[1], generator=torch.Generator().manual_seed(60 + i))
            one = dict(one, pts=one["pts"][:, perm].contiguous())
        parts.append(one)
    return kw, parts


@pytest.mark.parametrize("variant", routes.VARIANTS)
@pytest.mark.parametrize("permuted", [False, True], ids=["bin_route", "gaussian_route"])
def test_sample_alone_equals_sample_in_batch(variant, permuted):
    kw, parts = _three(variant, permuted)
    batch = {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}
    m = h.make_module(kw, variant)
    with deterministic():
        t = h.to_dev(batch, requires_grad=True)
        outs = routes._outputs(m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
        g, dev = routes._upstream(outs, 11)
        torch.autograd.backward(list(outs), dev)
        for b in range(3):
            one = h.to_dev(parts[b], requires_grad=True)
            o1 = routes._outputs(m(one["pts"], one["means"], one["opa"], one["sem"], one["scales"], one["cov"]))
            torch.autograd.backward(list(o1), [x[b].cuda() for x in g])
            for k in GRADS:
                diff = int((_bits(one[k].grad[0]) != _bits(t[k].grad[b])).sum())
                assert diff == 0, f"{variant} sample {b}: grad {k} alone vs in the batch differs in {diff} entries"


# ------------------------------------------------------------------------------------------------ hooks
def _route_words(kw, inp, variant):
    """one deterministic backward through splat_backward_raw with our own workspace; its route word per sample
    (``inp["pts"]`` [N, 3]: one point array shared by the batch)"""
    from gaussianformer_b200.splat import _desc_for, splat_backward_raw, splat_forward_raw
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    B, G = t["means"].shape[:2]
    desc = _desc_for(m._cfg(), B, G, t["pts"].shape[-2], t["sem"].shape[-1], t["pts"].dim() == 2)
    cov = t["cov"].reshape(B, G, 9).contiguous()
    (lg, bl, de, pr), _ = splat_forward_raw(desc, t["pts"], t["means"], t["opa"], t["sem"], cov, scales=t["scales"])
    gen = torch.Generator(device="cuda").manual_seed(3)
    prob = variant != "base"
    g = (torch.randn(lg.shape, device="cuda", generator=gen), torch.randn(bl.shape, device="cuda", generator=gen) if prob else None,
         torch.randn(bl.shape, device="cuda", generator=gen) if prob else None)
    L = _lib.lib()
    ws = torch.empty(L.gf_splat_backward_workspace_bytes_ex(ctypes.byref(desc), _lib.GF_BWD_DETERMINISTIC),
                     dtype=torch.uint8, device="cuda")
    splat_backward_raw(desc, t["pts"], t["means"], t["opa"], t["sem"], cov, g, (lg, bl, pr) if prob else (None,) * 3,
                       scales=t["scales"], deterministic=True, workspace=ws)
    words = (ctypes.c_uint32 * B)()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.gf_debug_splat_backward_route(ctypes.byref(desc), ctypes.c_void_p(ws.data_ptr()), stream, words))
    return list(words)


@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_route_words(variant):
    kw, inp = routes._case(variant)
    assert _route_words(kw, inp, variant) == [_lib.GF_DEBUG_ROUTE_BIN]
    kw, inp, _ = routes._route_inputs(variant, "permuted")
    assert _route_words(kw, inp, variant) == [_lib.GF_DEBUG_ROUTE_STRAY_POINTS]
    kw, inp, _ = routes._route_inputs(variant, "subset_dups")
    assert _route_words(kw, inp, variant) == [_lib.GF_DEBUG_ROUTE_GAUSSIAN]
    kw, inp = routes._mixed_batch(variant)
    assert _route_words(kw, inp, variant) == [_lib.GF_DEBUG_ROUTE_BIN, _lib.GF_DEBUG_ROUTE_STRAY_POINTS]


@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_slot_overflow_hands_over(variant):
    kw, inp = routes._case(variant)
    with plan(slot_budget=1):
        assert _route_words(kw, inp, variant) == [_lib.GF_DEBUG_ROUTE_SLOT_OVERFLOW]
        with deterministic():
            routes._check_vs_oracle(kw, inp, variant, f"{variant}/slot overflow", big_box=())
            _repeatable(kw, inp, variant, f"{variant}/slot overflow")


@pytest.mark.parametrize("variant", routes.VARIANTS)
@pytest.mark.parametrize("route", ["canonical", "permuted", "subset_dups"])
def test_sm_count_does_not_change_the_bytes(variant, route):
    kw, inp, offset, _ = _matrix_inputs(variant, route)
    with deterministic():
        ref = _grads(kw, inp, variant, offset=offset)
        for sms in (7, 1, 264):
            with plan(num_sms=sms):
                _assert_same_bits([ref, _grads(kw, inp, variant, offset=offset)], f"{variant}/{route} with {sms} SMs")


# ------------------------------------------------------------------------------------------------ switch off
def test_switch_off_runs_todays_kernels():
    seen_off, seen_on = set(), set()
    for variant in routes.VARIANTS:
        for route in ("canonical", "permuted", "subset_dups"):
            kw, inp, offset, _ = _matrix_inputs(variant, route)
            for on, seen in ((False, seen_off), (True, seen_on)):
                with deterministic(on):
                    names = routes._kernel_names(routes._fwd_bwd(kw, inp, variant, offset))
                seen |= names
                new = sorted(n for n in names if any(k in n for k in NEW_KERNELS))
                if not on:
                    assert not new, f"{variant}/{route} with the switch off ran {new}"
                    assert any("backward_small_kernel" in n for n in names), (variant, route)
                else:
                    assert new, f"{variant}/{route} with the switch on ran no deterministic kernel"
    assert any("backward_bin_kernel" in n for n in seen_off) and any("bin_finish_kernel" in n for n in seen_off)
    for k in NEW_KERNELS:
        assert any(k in n for n in seen_on), f"no route ran {k}"


# ------------------------------------------------------------------------------------------------ deformable aggregation
def _daf_runs():
    from gaussianformer_b200.ops import DeformableAggregationFunction as DAF
    from gaussianformer_b200.ops import deformable_aggregation_fused
    from gaussianformer_b200.synthetic import make_daf_fused_inputs, make_daf_inputs

    def plain():
        fms, loc, w = make_daf_inputs(num_anchor=16, num_pts=3, batch=1, num_cams=2, embed_dims=128, num_groups=4,
                                      levels=((6, 8), (3, 4)), visible_p=0.5, seed=3)
        feat, shape, start = DAF.feature_maps_format([f.cuda() for f in fms])
        feat = feat.contiguous().requires_grad_()
        return DAF.apply(feat, shape, start, loc.cuda().requires_grad_(), w.cuda().requires_grad_())

    def fused():
        fms, loc, logits, pm, wm = make_daf_fused_inputs(num_anchor=8, num_pts=3, batch=1, num_cams=2, embed_dims=128,
                                                         num_groups=4, levels=((6, 8), (3, 4)), visible_p=0.5, seed=21,
                                                         attn_drop=0.15)
        feat, shape, start = DAF.feature_maps_format([f.cuda() for f in fms])
        feat = feat.contiguous().requires_grad_()
        return deformable_aggregation_fused(feat, shape, start, loc.cuda().requires_grad_(),
                                            logits.cuda().requires_grad_(), pm.cuda(), wm.cuda())
    return {"DeformableAggregationFunction.backward": plain, "deformable_aggregation_fused backward": fused}


@pytest.mark.parametrize("name", list(_daf_runs()))
def test_daf_backward_alerts(name):
    run = _daf_runs()[name]
    with deterministic():
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            out = run()                                   # the forward (and feature_maps_format) stay silent
        with pytest.raises(RuntimeError, match=f"{name} does not have a deterministic implementation"):
            out.sum().backward()
    with deterministic(warn_only=True):
        out = run()
        with pytest.warns(UserWarning, match=f"{name} does not have a deterministic implementation"):
            out.sum().backward()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        run().sum().backward()                            # switch off: silent
