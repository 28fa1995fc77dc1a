"""The splat and sampling ops under CUDA-graph replay and on reused buffers, against eager calls and the fp64 oracle.

A replay differs from an eager call in three ways: the host decisions (kernel selection, grids, tensor maps, the slot
budget of the deterministic route) are frozen at capture, while the device-side routes (stray points, slot overflow,
the big-box queue) must still switch inside the graph; every replay runs on the workspace the previous one left behind;
and every host-side CUDA call of the op must be capturable.  The captures follow PyTorch's recipe (eager warm-up on a
side stream, static inputs, upstream gradients and labels, a new input set ``copy_``-ed in before each replay).

Gates per replay: forward outputs and deterministic-mode gradients bit-identical to an eager call on the same inputs
(that eager call through the oracle gate of test_splat_routes_gpu); atomic-mode gradients against the fp64 oracle with
helpers.check_module_grads; the sampling ops' forward bit-identical to eager and their gradients against
oracle.daf_* / oracle.daf_fused_* with helpers.assert_grad_parity.

The last part runs the paths the NaN fill of torch.use_deterministic_algorithms never reached on poisoned outputs: the
atomic splat backward (raw ABI, deterministic=False, inside the switch) and the fused sampling op (warn_only), so an
entry a kernel fails to store shows up as a NaN instead of whatever the caching allocator handed back."""
import ctypes
import types
import warnings

import numpy as np
import pytest
import torch

import helpers as h
import oracle
import test_splat_routes_gpu as routes
from test_daf_half_gpu import assert_half_grad
from test_splat_deterministic_gpu import _bits, deterministic, plan
from gaussianformer_b200 import _lib

pytestmark = pytest.mark.gpu

MODES = ["atomic", "deterministic"]
GRADS = ("means", "opa", "sem", "cov")
SRT_GRADS = ("means", "opa", "sem", "scales", "rot")
BIN_EDGES = np.array([8, 4, 16])   # common.cuh kBinX, kBinY, kBinZ: the bins of the deterministic slot plan
COV_LOWER = [3, 6, 7]             # entries of the 3x3 layout below the diagonal: their gradient is exactly 0


def _mode(mode):
    return deterministic(mode == "deterministic")


def _same(a, b):
    """bitwise equality of two tensors of any dtype"""
    a, b = a.detach().contiguous(), b.detach().contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _assert_same(a, b, what):
    assert _same(a, b), f"{what}: not bit-identical ({int((a.detach() != b.detach()).sum())} entries differ)"


def _capture(fn):
    """PyTorch's recipe: one eager warm-up call on a side stream, then ``fn`` captured; returns (graph, its outputs)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    torch.cuda.synchronize()
    return g, out


def _load(static, values):
    with torch.no_grad():
        for k, v in values.items():
            static[k].copy_(v)


def _enlarged(inp, k=1.5):
    """the same Gaussians with every scale times k (and the inverse covariance to match): larger clipped boxes"""
    out = dict(inp, scales=inp["scales"] * k)
    if "cov" in out:
        out["cov"] = inp["cov"] / (k * k)
    return out


def _permuted(inp, seed=5):
    perm = torch.randperm(inp["pts"].shape[1], generator=torch.Generator().manual_seed(seed))
    return dict(inp, pts=inp["pts"][:, perm].contiguous())


def _big_boxes(kw, inp, variant):
    return int((routes._clipped_box_volumes(kw, inp, variant) > routes.K_BIG_BOX).sum())


def _bin_rows(kw, inp, variant):
    """rows of the deterministic slot plan: for each clipped box the 8x4x16 bins it overlaps, summed over the Gaussians"""
    _, _, mi, radii, _, dims = h.oracle_prep(kw, inp, variant)
    r = radii.reshape(len(mi), -1)
    lo = np.maximum(mi - r, 0)
    hi = np.minimum(mi + r, np.asarray(dims) - 1)
    nb = np.where((hi >= lo).all(1, keepdims=True), hi // BIN_EDGES - lo // BIN_EDGES + 1, 0)
    return int(np.prod(nb, axis=1).sum())


def _no_nan(x, what):
    bad = int(torch.isnan(x.detach()).sum())
    assert bad == 0, f"{what}: {bad} NaN entries (an entry the kernel never stored)"


# ------------------------------------------------------------------------------------------------ oracle gates
def _gate_outputs(outs, kw, inp, variant, what):
    """every sample's forward outputs against the fp64 oracle (test_splat_routes_gpu's gate)"""
    B = inp["means"].shape[0]
    for b in range(B):
        one = {k: v[b:b + 1] for k, v in inp.items()}
        mine = [o[b] if B > 1 else o for o in outs]
        for o in mine:
            _no_nan(o, f"{what} sample {b} output")
        routes._check_forward(mine, h.oracle_forward(kw, one, variant), variant, f"{what} sample {b}")


def _gate_grads(holder, outs, kw, inp, variant, up, what):
    """every sample's four gradients (``holder[k].grad``) against the fp64 oracle (helpers.check_module_grads)"""
    B = inp["means"].shape[0]
    for k in GRADS:
        _no_nan(holder[k].grad, f"{what} grad {k}")
    for b in range(B):
        one = {k: v[b:b + 1] for k, v in inp.items()}
        pick = (lambda x: x[b]) if B > 1 else (lambda x: x)
        mine = [pick(o) for o in outs]
        h.check_module_grads(holder, kw, one, variant, tuple(pick(x).numpy() for x in up), what=f"{what} sample {b}",
                             saved_from=routes._saved(mine, kw, one, variant), sample=b)


def _srt_cov(inp):
    from gaussianformer_b200.splat import inverse_covariance_from_srt
    return inverse_covariance_from_srt(inp["scales"].double(), inp["rot"].double()).float()


def _gate_srt(outs, scales_grad, rot_grad, kw, inp, variant, up, what):
    """forward_from_srt (B = 1): outputs and the scales / rotations gradients gated like
    test_splat_routes_gpu.test_forward_from_srt_generic_route"""
    from gaussianformer_b200.splat import inverse_covariance_from_srt
    ref_inp = {k: v for k, v in inp.items() if k != "rot"}
    ref_inp["cov"] = _srt_cov(inp)
    for o in outs:
        _no_nan(o, f"{what} output")
    routes._check_forward(outs, h.oracle_forward(kw, ref_inp, variant), variant, what, rtol=1e-3, atol=1e-4)
    g64, _ = h.oracle_grads(kw, ref_inp, variant, tuple(x.numpy() for x in up), routes._saved(outs, kw, ref_inp, variant))
    s64 = inp["scales"][0].double().requires_grad_(True)
    r64 = inp["rot"][0].double().requires_grad_(True)
    ref_s, ref_r = torch.autograd.grad(inverse_covariance_from_srt(s64, r64), (s64, r64),
                                       torch.from_numpy(np.asarray(g64["cov"], np.float64)))
    for name, mine, want in (("scales", scales_grad[0], ref_s), ("rotations", rot_grad[0], ref_r)):
        _no_nan(mine, f"{what} grad {name}")
        want = want.numpy()
        h.assert_close(mine.cpu().numpy(), want, rtol=2e-3, atol=2e-4 * max(1.0, float(np.abs(want).max())),
                       what=f"{what} grad {name}")


# ------------------------------------------------------------------------------------------------ module steps
def _to_dev(inp, leaves):
    t = {k: v.cuda() for k, v in inp.items()}
    for k in leaves:
        t[k].requires_grad_(True)
    return t


def _module_call(m, t):
    return routes._outputs(m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))


def _srt_call(m, t):
    return routes._outputs(m.forward_from_srt(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["rot"]))


def _eager(kw, variant, inp, mode, up, call=_module_call, leaves=GRADS):
    """one eager forward + backward on fresh tensors: (outputs, leaf tensors holding their .grad)"""
    m = h.make_module(kw, variant)
    t = _to_dev(inp, leaves)
    with _mode(mode):
        outs = call(m, t)
        torch.autograd.backward(list(outs), [u.cuda() for u in up])
    return [o.detach() for o in outs], t


class _GraphStep:
    """module forward + torch.autograd.backward captured as one graph on static inputs and upstream gradients"""

    def __init__(self, kw, variant, inp, mode, call=_module_call, leaves=GRADS):
        self.kw, self.variant, self.mode, self.call, self.leaves = kw, variant, mode, call, leaves
        self.m = h.make_module(kw, variant, validate=False)      # no status-word read: nothing syncs inside the step
        self.t = _to_dev(inp, leaves)
        with _mode(mode):
            shapes = [o.shape for o in call(self.m, self.t)]
        self.up = [torch.zeros(s, device="cuda") for s in shapes]

        def step():
            for k in leaves:
                self.t[k].grad = None
            outs = call(self.m, self.t)
            torch.autograd.backward(list(outs), self.up)
            return [o.detach() for o in outs]

        with _mode(mode):
            self.graph, self.outs = _capture(step)

    def replay(self, inp, seed):
        """replay on ``inp`` with the upstream gradients of ``seed``; returns them (CPU)"""
        up, _ = routes._upstream(self.outs, seed)
        _load(self.t, inp)
        for u, c in zip(self.up, up):
            u.copy_(c)
        self.graph.replay()
        torch.cuda.synchronize()
        return up

    def bits(self):
        return [_bits(o) for o in self.outs], {k: _bits(self.t[k].grad) for k in self.leaves}

    def check(self, inp, seed, what, oracle_gate=True):
        """replay on ``inp``, then the gates: outputs (and deterministic gradients) == an eager call, bit for bit;
        atomic gradients against the oracle.  Returns the replay's bits."""
        up = self.replay(inp, seed)
        outs, t = _eager(self.kw, self.variant, inp, self.mode, up, self.call, self.leaves)
        for i, (a, b) in enumerate(zip(self.outs, outs)):
            _assert_same(a, b, f"{what}: graph output {i} vs eager")
        if self.mode == "deterministic":
            for k in self.leaves:
                _assert_same(self.t[k].grad, t[k].grad, f"{what}: graph grad {k} vs eager")
        holder = t if self.mode == "deterministic" else self.t     # the gradients the oracle sees
        if not (oracle_gate or self.mode == "atomic"):
            return self.bits()
        if self.call is _srt_call:
            _gate_srt([o.cpu() for o in outs], holder["scales"].grad, holder["rot"].grad, self.kw, inp, self.variant,
                      up, what)
        else:
            _gate_outputs([o.cpu() for o in outs], self.kw, inp, self.variant, what)
            _gate_grads(holder, [o.cpu() for o in outs], self.kw, inp, self.variant, up, what)
        return self.bits()


def _step_sets(variant):
    """(kw, capture set, replay sets): other Gaussians; the same with permuted points (stray points in the render, the
    bin kernel's hand-over to the Gaussian-centric chain); scales times ENLARGE (more clipped boxes above kBigBox than
    at capture); the first set again"""
    kw, cap = routes._case(variant)
    _, other = routes._case(variant, seed=routes.BASE_INPUTS[variant][1] + 20)
    big = _enlarged(other, ENLARGE[variant])
    assert _big_boxes(kw, big, variant) > _big_boxes(kw, cap, variant)
    return kw, cap, [other, _permuted(other), big, other]


# scale factor per variant that puts more clipped boxes above kBigBox than the capture set has (the base case's boxes
# are at most 13 x 13 x 4 voxels, apart from the whole-grid Gaussian)
ENLARGE = {"base": 3.0, "prob": 1.5, "prob_fast": 1.5}


SEEDS = [7, 8, 9, 7]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_whole_step_graph(variant, mode):
    kw, cap, sets = _step_sets(variant)
    step = _GraphStep(kw, variant, cap, mode)
    names = ["other Gaussians", "permuted points", "enlarged scales", "first set again"]
    runs = [step.check(inp, seed, f"{variant}/{mode} replay {i} ({names[i]})", oracle_gate=i < 3)
            for i, (inp, seed) in enumerate(zip(sets, SEEDS))]
    (o0, g0), (o3, g3) = runs[0], runs[3]
    for i, (a, b) in enumerate(zip(o0, o3)):
        assert torch.equal(a, b), f"{variant}/{mode}: output {i} of the repeated set differs from the first replay"
    if mode == "deterministic":
        for k in GRADS:
            assert torch.equal(g0[k], g3[k]), f"{variant}/{mode}: grad {k} of the repeated set differs from the first replay"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_mixed_batch_graph(variant, mode):
    """B = 2, captured on two canonical samples; replayed with one sample permuted (per-sample routes in one launch)"""
    kw, mixed = routes._mixed_batch(variant)
    _, b = routes._case(variant)
    cap = {k: torch.cat([mixed[k][:1], b[k]], 0) for k in mixed}            # both canonical
    swapped = {k: torch.cat([mixed[k][1:], mixed[k][:1]], 0) for k in mixed}  # permuted sample first
    step = _GraphStep(kw, variant, cap, mode)
    step.check(mixed, 3, f"{variant}/{mode} mixed batch")
    step.check(swapped, 4, f"{variant}/{mode} swapped mixed batch")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_forward_from_srt_graph(variant, mode):
    kw, inp = routes._case(variant)
    G = inp["means"].shape[1]
    gen = torch.Generator().manual_seed(23)
    cap = {k: v for k, v in inp.items() if k != "cov"}
    cap["rot"] = torch.randn(1, G, 4, generator=gen) * 1.5
    _, other = routes._case(variant, seed=routes.BASE_INPUTS[variant][1] + 20)
    other = {k: v for k, v in other.items() if k != "cov"}
    other["rot"] = torch.randn(1, G, 4, generator=gen) * 1.5
    step = _GraphStep(kw, variant, cap, mode, call=_srt_call, leaves=SRT_GRADS)
    first = step.check(_permuted(cap, 23), 29, f"{variant}/{mode} srt permuted")
    step.check(other, 30, f"{variant}/{mode} srt other Gaussians")
    again = step.check(_permuted(cap, 23), 29, f"{variant}/{mode} srt permuted again", oracle_gate=False)
    assert all(torch.equal(a, b) for a, b in zip(first[0], again[0])), f"{variant}/{mode} srt: repeated outputs differ"


# ------------------------------------------------------------------------------------------------ raw ABI helpers
def _raw_dev(kw, variant, inp, m):
    from gaussianformer_b200.splat import _desc_for
    t = {k: v.cuda().contiguous() for k, v in inp.items()}
    B, G = t["means"].shape[:2]
    if "cov" in t:
        t["cov"] = t["cov"].reshape(B, G, 9).contiguous()
    desc = _desc_for(m._cfg(), B, G, t["pts"].shape[1], t["sem"].shape[-1], False)
    return desc, t


def _raw_forward(desc, t):
    from gaussianformer_b200.splat import splat_forward_raw
    (lg, bl, de, pr), ws = splat_forward_raw(desc, t["pts"], t["means"], t["opa"], t["sem"], t.get("cov"),
                                             scales=t["scales"], rotations=t.get("rot"))
    return (lg, bl, de, pr), ws


def _raw_backward(desc, t, fwd, up, prob, ws, det):
    from gaussianformer_b200.splat import splat_backward_raw
    lg, bl, de, pr = fwd
    grads_in = (up[0], up[1] if prob else None, up[2] if prob else None)
    saved = (lg, bl, pr) if prob else (None,) * 3
    return splat_backward_raw(desc, t["pts"], t["means"], t["opa"], t["sem"], t.get("cov"), grads_in, saved,
                              scales=t["scales"], rotations=t.get("rot"), deterministic=det, workspace=ws)


def _bwd_ws(desc, det):
    L = _lib.lib()
    n = L.gf_splat_backward_workspace_bytes_ex(ctypes.byref(desc), _lib.GF_BWD_DETERMINISTIC if det else 0)
    return torch.empty(max(n, 256), dtype=torch.uint8, device="cuda")


def _route_words(desc, ws):
    words = (ctypes.c_uint32 * max(int(desc.batch), 1))()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib().gf_debug_splat_backward_route(ctypes.byref(desc), ctypes.c_void_p(ws.data_ptr()), stream, words))
    return list(words)


def _raw_up(desc, prob, seed):
    B, N, C = max(int(desc.batch), 1), desc.N, desc.C
    gen = torch.Generator().manual_seed(seed)
    up = [torch.randn(B, N, C, generator=gen)]
    if prob:
        up += [torch.randn(B, N, generator=gen), torch.randn(B, N, generator=gen)]
    return up


def _raw_gate(grads, fwd, kw, inp, variant, up, what):
    """raw-ABI gradients (g_means, g_opa, g_sem, g_cov [B,G,9]) of every sample against the oracle; no NaN, the
    cov gradient's lower triangle exactly 0"""
    gm, go, gs, gc = grads[:4]
    B, G = gm.shape[:2]
    holder = {}
    for k, x in zip(GRADS, (gm, go, gs, gc.view(B, G, 3, 3))):
        _no_nan(x, f"{what} grad {k}")
        holder[k] = types.SimpleNamespace(grad=x)
    lower = gc.reshape(B, G, 9)[..., COV_LOWER]
    assert torch.equal(lower, torch.zeros_like(lower)), f"{what}: cov gradient below the diagonal is not exactly 0"
    outs = [x.cpu() for x in fwd[:3] if x is not None] if variant != "base" else [fwd[0].cpu()]
    if B == 1:
        outs = [o[0] for o in outs]
    _gate_grads(holder, outs, kw, inp, variant, [u if B > 1 else u[0] for u in up], what)


# ------------------------------------------------------------------------------------------------ slot overflow in a graph
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_slot_overflow_inside_a_frozen_graph(variant):
    """slot budget R = set A's row count, frozen at capture: set A fits (bin route), set B (scales x 1.5) overflows and
    the graph's own slot plan hands it to the Gaussian-centric chain; both equal eager calls under the same budget"""
    kw, a = routes._case(variant)
    b = _enlarged(a)
    R = _bin_rows(kw, a, variant)
    assert _bin_rows(kw, b, variant) > R
    prob = variant != "base"
    m = h.make_module(kw, variant, validate=False)
    desc, t = _raw_dev(kw, variant, a, m)
    up = [u.cuda() for u in _raw_up(desc, prob, 3)]
    with plan(slot_budget=R):
        ws = _bwd_ws(desc, True)

        def step():
            fwd, _ = _raw_forward(desc, t)
            return fwd, _raw_backward(desc, t, fwd, up, prob, ws, True)

        graph, (g_fwd, g_grads) = _capture(step)
    for name, inp, seed, word in (("A", a, 3, _lib.GF_DEBUG_ROUTE_BIN), ("B", b, 4, _lib.GF_DEBUG_ROUTE_SLOT_OVERFLOW)):
        _, dev = _raw_dev(kw, variant, inp, m)
        _load(t, dev)
        ups = _raw_up(desc, prob, seed)
        for u, c in zip(up, ups):
            u.copy_(c)
        graph.replay()
        torch.cuda.synchronize()
        assert _route_words(desc, ws) == [word], f"{variant} set {name}: route word {_route_words(desc, ws)}"
        with plan(slot_budget=R):          # the eager call under the same budget, on its own workspace
            ews = _bwd_ws(desc, True)
            e_fwd, _ = _raw_forward(desc, dev)
            e_grads = _raw_backward(desc, dev, e_fwd, [u.cuda() for u in ups], prob, ews, True)
            assert _route_words(desc, ews) == [word]
        for i, (x, y) in enumerate(zip(g_fwd, e_fwd)):
            if x is not None:
                _assert_same(x, y, f"{variant} set {name}: graph forward output {i} vs eager")
        for k, x, y in zip(GRADS, g_grads[:4], e_grads[:4]):
            _assert_same(x, y, f"{variant} set {name}: graph grad {k} vs eager")
        _raw_gate(e_grads, e_fwd, kw, inp, variant, ups, f"{variant} set {name} (eager, slot budget {R})")


# ------------------------------------------------------------------------------------------------ fused epilogue in a graph
def _eval_sets():
    sets = []
    for seeds in ((51, 52, 53), (61, 62, 63), (71, 72, 73)):
        parts = [h.splat_case("tiny", s, True)[1] for s in seeds]
        inp = {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}
        gen = torch.Generator().manual_seed(seeds[0])
        B, N = inp["pts"].shape[:2]
        labels = torch.randint(0, 18, (B, N), generator=gen)
        labels[torch.rand(B, N, generator=gen) < 0.2] = 255
        sets.append((inp, labels.to(torch.uint8)))
    return h.splat_case("tiny", 51, True)[0], sets


def test_forward_eval_and_on_grid_graph():
    kw, sets = _eval_sets()
    m = h.make_module(kw, "base", validate=False)
    t = {k: v.cuda() for k, v in sets[0][0].items()}
    lab = sets[0][1].cuda()
    cw = (torch.rand(18, generator=torch.Generator().manual_seed(9)) + 0.5).cuda()
    g_eval, r = _capture(lambda: m.forward_eval(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"],
                                                labels=lab, class_weights=cw, layout="cn"))
    with torch.no_grad():
        g_grid, grid_logits = _capture(lambda: m.forward_on_grid(t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
    for i, (inp, labels) in enumerate(sets[1:] + sets[:1]):
        _load(t, {k: v.cuda() for k, v in inp.items()})
        lab.copy_(labels)
        g_eval.replay()
        g_grid.replay()
        torch.cuda.synchronize()
        e = {k: v.cuda() for k, v in inp.items()}
        ref = m.forward_eval(e["pts"], e["means"], e["opa"], e["sem"], e["scales"], e["cov"], labels=labels.cuda(),
                             class_weights=cw, layout="cn")
        _assert_same(r["pred_occ"], ref["pred_occ"], f"replay {i} pred_occ")
        _assert_same(r["final_occ"], ref["final_occ"], f"replay {i} final_occ")
        with torch.no_grad():
            logits = m(e["pts"], e["means"], e["opa"], e["sem"], e["scales"], e["cov"])
            _assert_same(grid_logits, m.forward_on_grid(e["means"], e["opa"], e["sem"], e["scales"], e["cov"]),
                         f"replay {i} forward_on_grid logits")
        want = torch.nn.functional.cross_entropy(logits.double().transpose(1, 2), labels.cuda().long(),
                                                 weight=cw.double(), ignore_index=255, reduction="mean")
        got = float(r["ce_loss"])
        assert abs(got - float(want)) <= 2e-5 * abs(float(want)) + 1e-6, (i, got, float(want))
        if i == 0:   # the eager op through the oracle gate
            one = {k: v[:1] for k, v in inp.items()}
            _assert_same(ref["pred_occ"][0].t(), logits[0], "forward_eval vs forward")
            routes._check_forward([logits[0].cpu()], h.oracle_forward(kw, one, "base"), "base", "forward_eval sample 0")
            grid_one = dict(one, pts=m.grid_points("cuda").cpu())
            routes._check_forward([grid_logits[0].cpu()], h.oracle_forward(kw, grid_one, "base"), "base",
                                  "forward_on_grid sample 0")


# ------------------------------------------------------------------------------------------------ bench recipe, full size
def test_bench_recipe_full_size_forward():
    """cfg 2: two resident sets, raw-ABI forward, one graph each, replayed interleaved"""
    sets = [h.splat_case("gs25600_solid", s, False) for s in (0, 1)]
    kw = sets[0][0]
    m = h.make_module(kw, "base", validate=False)
    graphs = []
    for _, inp, _ in sets:
        desc, t = _raw_dev(kw, "base", inp, m)
        graphs.append((_capture(lambda desc=desc, t=t: _raw_forward(desc, t)[0][0]), t))
    mv = h.make_module(kw, "base")
    eager = []
    for _, inp, _ in sets:
        t = h.to_dev(inp)
        with torch.no_grad():
            eager.append(mv(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
    ref = h.oracle_forward(kw, sets[0][1], "base")
    h.assert_close(eager[0].cpu().numpy(), ref["logits"], what="cfg2 eager logits")
    for order in ((0, 1), (1, 0), (0, 1)):
        for i in order:
            graphs[i][0][0].replay()
        torch.cuda.synchronize()
        for i in (0, 1):
            _assert_same(graphs[i][0][1][0], eager[i], f"cfg2 set {i} graph logits (order {order})")


def test_bench_recipe_batch_of_four_deterministic():
    """cfg 5 shape: 4 samples of cfg 2 in one batched call, module forward + backward captured in deterministic mode"""
    def batch(seeds):
        parts = [h.splat_case("gs25600_solid", s, False) for s in seeds]
        return parts[0][0], {k: torch.cat([p[1][k] for p in parts], 0) for k in parts[0][1]}
    kw, cap = batch((10, 11, 12, 13))
    step = _GraphStep(kw, "base", cap, "deterministic")
    for i, seeds in enumerate(((20, 21, 22, 23), (10, 11, 12, 13))):
        _, inp = batch(seeds)
        up = step.replay(inp, 40 + i)
        outs, t = _eager(kw, "base", inp, "deterministic", up)
        _assert_same(step.outs[0], outs[0], f"cfg5 replay {i} logits")
        for k in GRADS:
            _assert_same(step.t[k].grad, t[k].grad, f"cfg5 replay {i} grad {k}")


# ------------------------------------------------------------------------------------------------ make_graphed_callables
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", ["base", "prob"])
def test_make_graphed_callables(variant, mode):
    """forward and backward as two graphs; the backward graph runs in a later autograd call"""
    kw, cap, sets = _step_sets(variant)
    m = h.make_module(kw, variant, validate=False)
    t0 = _to_dev(cap, GRADS)
    args = tuple(t0[k] for k in ("pts", "means", "opa", "sem", "scales", "cov"))
    with _mode(mode):
        graphed = torch.cuda.make_graphed_callables(m, args)
    first = None
    for i, (inp, seed) in enumerate(zip(sets, SEEDS)):
        what = f"{variant}/{mode} graphed replay {i}"
        t = _to_dev(inp, GRADS)
        with _mode(mode):
            outs = routes._outputs(graphed(*(t[k] for k in ("pts", "means", "opa", "sem", "scales", "cov"))))
            outs = [o.clone() for o in outs]       # the graph's static outputs: the next replay overwrites them
        up, _ = routes._upstream(outs, seed)
        e_outs, e_t = _eager(kw, variant, inp, mode, up)           # between the forward and its backward
        for j, (a, b) in enumerate(zip(outs, e_outs)):
            _assert_same(a, b, f"{what}: output {j} vs eager")
        with _mode(mode):
            torch.autograd.backward(list(outs), [u.cuda() for u in up])
        grads = {k: t[k].grad.clone() for k in GRADS}
        holder = {k: types.SimpleNamespace(grad=grads[k]) for k in GRADS}
        if mode == "deterministic":
            for k in GRADS:
                _assert_same(grads[k], e_t[k].grad, f"{what}: grad {k} vs eager")
        if i < 3 and (mode == "atomic" or i == 0):
            cpu = [o.cpu() for o in e_outs]
            _gate_outputs(cpu, kw, inp, variant, what)
            _gate_grads(holder, cpu, kw, inp, variant, up, what)
        if i == 0:
            first = (outs, grads)
        elif i == 3:
            assert all(_same(a, b) for a, b in zip(first[0], outs)), f"{what}: outputs differ from replay 0"
            if mode == "deterministic":
                assert all(_same(first[1][k], grads[k]) for k in GRADS), f"{what}: grads differ from replay 0"


# ------------------------------------------------------------------------------------------------ sampling ops in a graph
DAF_SHAPES = {   # (embed, groups, levels, cameras): test_daf_gpu's shapes
    "fast": (128, 4, ((12, 20), (6, 10), (3, 5)), 3),
    "general": (16, 4, ((7, 12), (4, 6), (2, 3)), 3),
}
FUSED_SHAPES = {
    "one_slice": (128, 4, ((12, 20), (6, 10), (3, 5))),
    "two_slices": (256, 8, ((9, 7), (5, 4))),          # two channel slices per warp, 8 groups
}
HALF = {"f32": torch.float32, "f16": torch.float16}
K_PTS = 5


def _edge_locations(loc, weights=None):
    """a NaN location, a key point no camera sees; with ``weights`` [B,P,M,L,Gr]: an anchor whose weights are all 0
    and a group dropped for a whole anchor"""
    loc[1, 4, 2] = torch.tensor([float("nan"), 0.5])
    loc[0, 7] = 1.5
    if weights is not None:
        weights[1, 2 * K_PTS:3 * K_PTS] = 0
        weights[0, 4 * K_PTS:5 * K_PTS, :, :, 0] = 0


def _daf_set(shape, seed):
    embed, groups, levels, cams = DAF_SHAPES[shape]
    from gaussianformer_b200.synthetic import make_daf_inputs
    fms, loc, w = make_daf_inputs(num_anchor=16, num_pts=K_PTS, batch=2, num_cams=cams, embed_dims=embed,
                                  num_groups=groups, levels=levels, visible_p=0.5, seed=seed)
    _edge_locations(loc, w)
    return fms, loc, w


def _fused_set(shape, seed):
    embed, groups, levels = FUSED_SHAPES[shape]
    from gaussianformer_b200.synthetic import make_daf_fused_inputs
    B, A, M = 2, 12, 3
    fms, loc, logits, pm, wm = make_daf_fused_inputs(num_anchor=A, num_pts=K_PTS, batch=B, num_cams=M,
                                                     embed_dims=embed, num_groups=groups, levels=levels, visible_p=0.5,
                                                     seed=seed, attn_drop=0.15)
    _edge_locations(loc)
    pm = ((loc > 0) & (loc < 1)).all(-1).reshape(B, A, K_PTS, M).contiguous()
    pm[0, 0] = False                                     # an anchor no camera sees
    wm[0, 1, :, :, :, 0] = False                         # a group with every entry dropped
    return fms, loc, logits, pm, wm


def _table(maps):
    """[B, M, C, h, w] maps -> the [B, M, F, C] table layout (the reference's reshape + cat + permute)"""
    B, M, C = maps[0].shape[:3]
    return torch.cat([x.reshape(B, M, C, -1) for x in maps], -1).permute(0, 1, 3, 2).contiguous()


def _feat_gate(mine, rf, rf32, dtype, what):
    _no_nan(mine, what)
    if dtype is torch.float32:
        h.assert_grad_parity(mine.cpu().numpy(), rf, rf32, what=what)
    else:
        assert_half_grad(mine, rf, rf32, dtype, what)


def _run_daf(op, maps, loc, third, masks, up):
    """feature_maps_format -> op forward + backward; (output, [map grads], loc grad, weights / logits grad)"""
    from gaussianformer_b200.ops import DeformableAggregationFunction as DAF
    from gaussianformer_b200.ops import deformable_aggregation_fused
    for x in list(maps) + [loc, third]:
        x.grad = None
    feat, shape, start = DAF.feature_maps_format(list(maps))
    if op == "plain":
        out = DAF.apply(feat, shape, start, loc, third)
    else:
        out = deformable_aggregation_fused(feat, shape, start, loc, third, *masks)
    out.backward(up)
    return out.detach(), [x.grad for x in maps], loc.grad, third.grad


@pytest.mark.parametrize("dtype", list(HALF))
@pytest.mark.parametrize("op,shape", [("plain", s) for s in DAF_SHAPES] + [("fused", s) for s in FUSED_SHAPES])
def test_sampling_op_graph(op, shape, dtype):
    dt = HALF[dtype]
    make = _daf_set if op == "plain" else _fused_set
    sets = [make(shape, seed) for seed in (3, 4, 5, 6)]

    def dev(s):
        fms, loc, third = s[0], s[1], s[2]
        maps = [f.to(dt).cuda().requires_grad_() for f in fms]
        masks = tuple(x.cuda() for x in s[3:])
        return maps, loc.cuda().requires_grad_(), third.cuda().requires_grad_(), masks

    maps, loc, third, masks = dev(sets[0])
    B, C = loc.shape[0], maps[0].shape[2]
    out_shape = (B, loc.shape[1], C) if op == "plain" else (B, third.shape[1], C)
    up = torch.zeros(out_shape, device="cuda")
    graph, (g_out, g_maps, g_loc, g_third) = _capture(lambda: _run_daf(op, maps, loc, third, masks, up))
    for i, s in enumerate(sets[1:]):
        what = f"{op}/{shape}/{dtype} replay {i}"
        n_maps, n_loc, n_third, n_masks = dev(s)
        g_up = torch.randn(out_shape, generator=torch.Generator().manual_seed(11 + i))
        with torch.no_grad():
            for x, y in zip(maps + [loc, third] + list(masks), n_maps + [n_loc, n_third] + list(n_masks)):
                x.copy_(y)
            up.copy_(g_up)
        graph.replay()
        torch.cuda.synchronize()
        e_out, e_maps, e_loc, e_third = _run_daf(op, n_maps, n_loc, n_third, n_masks, g_up.cuda())
        _assert_same(g_out, e_out, f"{what}: graph output vs eager")
        f_np = _table([x.detach() for x in n_maps]).float().cpu().numpy()
        from gaussianformer_b200.ops import DeformableAggregationFunction as DAF
        _, shp, st = DAF.feature_maps_format([x.detach() for x in n_maps])
        s_np, st_np = shp.cpu().numpy(), st.cpu().numpy()
        loc_np, third_np = s[1].numpy(), s[2].numpy()
        if op == "plain":
            ref = oracle.daf_forward(f_np, s_np, st_np, loc_np, third_np, "f64")
            r64 = oracle.daf_backward(f_np, s_np, st_np, loc_np, third_np, g_up.numpy(), "f64")
            r32 = oracle.daf_backward(f_np, s_np, st_np, loc_np, third_np, g_up.numpy(), "f32")
            names = ("weights", "loc")
            rf, rl, rt = r64
            rf32, rl32, rt32 = r32
        else:
            pm_np, wm_np = s[3].numpy(), s[4].numpy()
            ref = oracle.daf_fused_forward(f_np, s_np, st_np, loc_np, third_np, pm_np, wm_np, "f64")
            rf, rl, rt = oracle.daf_fused_backward(f_np, s_np, st_np, loc_np, third_np, g_up.numpy(), pm_np, wm_np, "f64")
            rf32, rl32, rt32 = oracle.daf_fused_backward(f_np, s_np, st_np, loc_np, third_np, g_up.numpy(), pm_np, wm_np,
                                                         "f32")
            names = ("logits", "loc")
            assert torch.all(g_out[0, 0] == 0) and torch.all(g_third[0, 0] == 0), f"{what}: unseen anchor not exactly 0"
        _no_nan(g_out, f"{what} output")
        h.assert_close(g_out.cpu().numpy(), ref, what=f"{what} output")
        _feat_gate(_table(g_maps), rf, rf32, dt, f"{what} grad feat")
        for name, mine, r, r_32 in ((names[0], g_third, rt, rt32), (names[1], g_loc, rl, rl32)):
            _no_nan(mine, f"{what} grad {name}")
            h.assert_grad_parity(mine.cpu().numpy(), r, r_32, what=f"{what} grad {name}")


# ------------------------------------------------------------------------------------------------ workspace reuse
def _forward_on(desc, t, ws, prob):
    """gf_splat_forward on a caller-owned workspace (splat_forward_raw allocates a fresh one per call)"""
    from gaussianformer_b200.splat import _ptr
    L = _lib.lib()
    B, N, C = max(int(desc.batch), 1), desc.N, desc.C
    lg = torch.empty((B, N, C), device="cuda")
    extra = [torch.empty((B, N), device="cuda") for _ in range(3)] if prob else [None] * 3
    ins = _lib.SplatInputs(_ptr(t["pts"]), None, _ptr(t["means"]), None, _ptr(t["opa"]), _ptr(t["sem"]),
                           _ptr(t["cov"]), None, _ptr(t["scales"]), None)
    outs = _lib.SplatOutputs(_ptr(lg), *(_ptr(x) for x in extra), None, None, None, None, None)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.gf_splat_forward(ctypes.byref(desc), ctypes.byref(ins), ctypes.byref(outs), _ptr(ws), ws.numel(), stream))
    return [lg] + [x for x in extra if x is not None]


@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_forward_workspace_left_by_a_failed_call(variant):
    """call A has a mean on the grid's upper face (status flags set); call B, valid, on the same workspace: its
    status word reads 0 and its outputs equal B on a fresh workspace"""
    from gaussianformer_b200.splat import read_flags
    kw, b = routes._case(variant)
    dims, gs, pc = (kw["H"], kw["W"], kw["D"]), kw["grid_size"], kw["pc_min"]
    a = dict(b, means=b["means"].clone())
    a["means"][0, 1, 0] = float(np.float32(dims[0]) * np.float32(gs) + np.float32(pc[0]))
    m = h.make_module(kw, variant)
    prob = variant != "base"
    desc, ta = _raw_dev(kw, variant, a, m)
    _, tb = _raw_dev(kw, variant, b, m)
    ws = torch.empty(_lib.lib().gf_splat_forward_workspace_bytes(ctypes.byref(desc)), dtype=torch.uint8, device="cuda")
    _forward_on(desc, ta, ws, prob)
    assert read_flags(ws, ws.device) & _lib.GF_FLAG_MEAN_OUT_OF_GRID
    outs = _forward_on(desc, tb, ws, prob)
    assert read_flags(ws, ws.device) == 0
    fresh = _forward_on(desc, tb, torch.empty_like(ws), prob)
    for i, (x, y) in enumerate(zip(outs, fresh)):
        _assert_same(x, y, f"{variant}: output {i} on the reused workspace vs a fresh one")
    _gate_outputs([o[0].cpu() for o in outs[:3]], kw, b, variant, f"{variant} reused forward workspace")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_backward_workspace_reused(variant, mode):
    """permuted -> canonical -> enlarged scales (more big boxes) -> canonical, all on one backward workspace"""
    det = mode == "deterministic"
    kw, canon = routes._case(variant)
    _, permuted, _ = routes._route_inputs(variant, "permuted")
    seq = [("permuted", permuted, _lib.GF_DEBUG_ROUTE_STRAY_POINTS), ("canonical", canon, _lib.GF_DEBUG_ROUTE_BIN),
           ("enlarged", _enlarged(canon), _lib.GF_DEBUG_ROUTE_BIN), ("canonical again", canon, _lib.GF_DEBUG_ROUTE_BIN)]
    prob = variant != "base"
    m = h.make_module(kw, variant)
    desc, _ = _raw_dev(kw, variant, canon, m)
    ws = _bwd_ws(desc, det)
    for i, (name, inp, word) in enumerate(seq):
        what = f"{variant}/{mode} {name} on a reused workspace"
        _, t = _raw_dev(kw, variant, inp, m)
        fwd, _ = _raw_forward(desc, t)
        up = _raw_up(desc, prob, 20 + i)
        grads = _raw_backward(desc, t, fwd, [u.cuda() for u in up], prob, ws, det)
        torch.cuda.synchronize()
        if det:
            assert _route_words(desc, ws) == [word], f"{what}: route word {_route_words(desc, ws)}, want {word}"
            fresh = _raw_backward(desc, t, fwd, [u.cuda() for u in up], prob, None, True)
            for k, x, y in zip(GRADS, grads[:4], fresh[:4]):
                _assert_same(x, y, f"{what}: grad {k} vs a fresh workspace")
        _raw_gate(grads, fwd, kw, inp, variant, up, what)


# ------------------------------------------------------------------------------------------------ poisoned outputs
def _assert_poisoning():
    """torch.use_deterministic_algorithms(True) fills torch.empty with NaN: inside the switch, every output the op
    allocates starts as NaN (the atomic backward is asked for explicitly, deterministic=False)"""
    assert torch.isnan(torch.empty(8, device="cuda")).all(), "torch.empty is not NaN-filled under the switch"


def _empty_box_inputs(variant):
    """subset_dups-style: every point inside one Gaussian's clipped box dropped (N != H*W*D); returns (kw, inp, g)"""
    kw, inp = routes._case(variant)
    _, _, mi, radii, _, dims = h.oracle_prep(kw, inp, variant)
    r = radii.reshape(len(mi), -1)
    lo = np.maximum(mi - r, 0)
    hi = np.minimum(mi + r, np.asarray(dims) - 1)
    vol = np.prod(np.maximum(hi - lo + 1, 0), axis=1)
    g = int(np.argsort(np.where(vol >= 8, vol, np.iinfo(np.int64).max))[0])
    vox = np.stack(np.unravel_index(np.arange(inp["pts"].shape[1]), dims), 1)   # canonical: point n in voxel n
    inside = ((vox >= lo[g]) & (vox <= hi[g])).all(1)
    keep = torch.from_numpy(np.nonzero(~inside)[0])
    assert inside.sum() == vol[g] and len(keep) > 0
    return kw, dict(inp, pts=inp["pts"][:, keep].contiguous()), g


def _poison_inputs(variant, route):
    if route == "canonical":
        return routes._case(variant) + (None,)
    if route == "mixed_batch":
        return routes._mixed_batch(variant) + (None,)
    if route == "empty_box":
        return _empty_box_inputs(variant)
    kw, inp, _ = routes._route_inputs(variant, route)
    return kw, inp, None


@pytest.mark.parametrize("route", ["canonical", "permuted", "subset_dups", "ragged", "mixed_batch", "empty_box"])
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_atomic_backward_on_poisoned_outputs(variant, route):
    kw, inp, empty_g = _poison_inputs(variant, route)
    prob = variant != "base"
    m = h.make_module(kw, variant)
    desc, t = _raw_dev(kw, variant, inp, m)
    fwd, _ = _raw_forward(desc, t)
    up = _raw_up(desc, prob, 13)
    ws = _bwd_ws(desc, False)
    with deterministic():
        _assert_poisoning()
        grads = _raw_backward(desc, t, fwd, [u.cuda() for u in up], prob, ws, False)
        torch.cuda.synchronize()
    _raw_gate(grads, fwd, kw, inp, variant, up, f"{variant}/{route} poisoned atomic backward")
    if empty_g is not None:
        for k, x in zip(GRADS, grads[:4]):
            assert torch.all(x[0, empty_g] == 0), f"{variant}: grad {k} of the Gaussian whose box holds no point " \
                                                  f"is not exactly 0: {x[0, empty_g]}"


@pytest.mark.parametrize("route", ["canonical", "permuted"])
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_atomic_srt_backward_on_poisoned_outputs(variant, route):
    kw, inp = routes._case(variant)
    if route == "permuted":
        inp = _permuted(inp, 23)
    inp = {k: v for k, v in inp.items() if k != "cov"}
    inp["rot"] = torch.randn(1, inp["means"].shape[1], 4, generator=torch.Generator().manual_seed(23)) * 1.5
    prob = variant != "base"
    m = h.make_module(kw, variant)
    desc, t = _raw_dev(kw, variant, inp, m)
    fwd, _ = _raw_forward(desc, t)
    up = _raw_up(desc, prob, 29)
    ws = _bwd_ws(desc, False)
    with deterministic():
        _assert_poisoning()
        gm, go, gs, gc, gsc, grot = _raw_backward(desc, t, fwd, [u.cuda() for u in up], prob, ws, False)
        torch.cuda.synchronize()
    assert gc is None
    what = f"{variant}/{route} poisoned srt backward"
    for k, x in (("means", gm), ("opa", go), ("sem", gs)):
        _no_nan(x, f"{what} grad {k}")
    outs = [x[0].cpu() for x in fwd[:3]] if prob else [fwd[0][0].cpu()]
    _gate_srt(outs, gsc, grot, kw, inp, variant, [u[0] for u in up], what)


@pytest.mark.parametrize("embed,groups,levels,masks", [
    (128, 4, ((12, 20), (6, 10), (3, 5)), "both"),
    (128, 4, ((12, 20), (6, 10), (3, 5)), "point"),
    (256, 8, ((9, 7), (5, 4)), "both"),
    (128, 1, ((5, 5),), "point"),
])
def test_fused_sampling_on_poisoned_outputs(embed, groups, levels, masks):
    """the masked cases of test_daf_gpu.test_daf_fused_forward_backward_vs_oracle with output, stats and grad_logits
    NaN-filled (warn_only: the backward warns instead of raising); exact zeros wherever the oracle's are zero"""
    from gaussianformer_b200.ops import DeformableAggregationFunction as DAF
    from gaussianformer_b200.ops import deformable_aggregation_fused
    from gaussianformer_b200.synthetic import make_daf_fused_inputs
    B, A, K, M = 2, 40, 5, 3
    fms, loc, logits, pm, wm = make_daf_fused_inputs(num_anchor=A, num_pts=K, batch=B, num_cams=M, embed_dims=embed,
                                                     num_groups=groups, levels=levels, visible_p=0.5, seed=21,
                                                     attn_drop=0.15)
    loc[0, 2, 0] = torch.tensor([0.004, 0.996]); loc[0, 3, 1] = torch.tensor([0.999, 0.001])
    loc[1, 4, 2] = torch.tensor([float("nan"), 0.5])
    pm = ((loc > 0) & (loc < 1)).all(-1).reshape(B, A, K, M).contiguous()
    pm[0, 0] = False
    wm[0, 1, :, :, :, 0] = False
    logits[1, 2, 0, 0, 0, 0] = 30.0
    if masks == "point":
        wm = None
    feat, shape, start = DAF.feature_maps_format([f.cuda() for f in fms])
    feat = feat.contiguous().requires_grad_()
    loc_d = loc.cuda().requires_grad_()
    lg_d = logits.cuda().requires_grad_()
    g = torch.randn(B, A, embed, generator=torch.Generator().manual_seed(5))
    with deterministic(warn_only=True), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _assert_poisoning()
        out = deformable_aggregation_fused(feat, shape, start, loc_d, lg_d, pm.cuda(), None if wm is None else wm.cuda())
        out.backward(g.cuda())
        torch.cuda.synchronize()
    f_np, s_np, st_np = feat.detach().cpu().numpy(), shape.cpu().numpy(), start.cpu().numpy()
    pm_np, wm_np = pm.numpy(), None if wm is None else wm.numpy()
    ref = oracle.daf_fused_forward(f_np, s_np, st_np, loc.numpy(), logits.numpy(), pm_np, wm_np, "f64")
    rf, rl, rw = oracle.daf_fused_backward(f_np, s_np, st_np, loc.numpy(), logits.numpy(), g.numpy(), pm_np, wm_np, "f64")
    rf32, rl32, rw32 = oracle.daf_fused_backward(f_np, s_np, st_np, loc.numpy(), logits.numpy(), g.numpy(), pm_np, wm_np,
                                                 "f32")
    for name, mine, r64, r32 in (("output", out.detach(), ref, None), ("grad feat", feat.grad, rf, rf32),
                                 ("grad logits", lg_d.grad, rw, rw32), ("grad loc", loc_d.grad, rl, rl32)):
        _no_nan(mine, f"poisoned fused {name}")
        x = mine.cpu().numpy()
        if r32 is None:
            h.assert_close(x, r64, what=f"poisoned fused {name}")
        else:
            h.assert_grad_parity(x, r64, r32, what=f"poisoned fused {name}")
        if name == "grad feat":
            continue
        zero = np.asarray(r64) == 0
        assert (x[zero] == 0).all(), f"poisoned fused {name}: {int((x[zero] != 0).sum())} entries not 0 where the oracle's are"
