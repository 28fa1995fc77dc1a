"""numpy oracle of the submanifold sparse convolution (include/gf_b200.h, gf_subm_conv_*) in fp64 or fp32: a dict voxel
lookup with the lowest-row representative, per-offset pair lists and matmuls, for the output and all three gradients.
Independent of the device code: no dense table, no scan, no sort."""
import numpy as np


def rulebook(indices, spatial, batch, k):
    """dict with valid [N] bool, slot [N] (-1 invalid), rep [M], voxels [M, 4], nbr [M, k^3] (slot or -1),
    pairs[o] = (dst slots, src slots) ascending in dst"""
    idx = np.asarray(indices, np.int64)
    X, Y, Z = spatial
    lim = np.array([batch, X, Y, Z])
    valid = ((idx >= 0) & (idx < lim)).all(1)
    lowest = {}
    for i in np.nonzero(valid)[0]:
        key = tuple(idx[i])
        if key not in lowest:
            lowest[key] = int(i)
    voxels = sorted(lowest)                     # (b, x, y, z) order = the flat voxel order
    slot_of = {v: s for s, v in enumerate(voxels)}
    slot = np.array([slot_of[tuple(r)] if ok else -1 for r, ok in zip(idx, valid)], np.int64)
    rep = np.array([lowest[v] for v in voxels], np.int64)
    p = (k - 1) // 2
    K = k ** 3
    vox = np.array(voxels, np.int64).reshape(-1, 4)
    key = ((vox[:, 0] * X + vox[:, 1]) * Y + vox[:, 2]) * Z + vox[:, 3]   # ascending, as the voxels are sorted
    nbr = np.full((len(voxels), K), -1, np.int64)
    for o in range(K):
        q = vox[:, 1:] + np.array([o // (k * k) - p, (o // k) % k - p, o % k - p])
        inside = ((q >= 0) & (q < np.array(spatial))).all(1)
        qk = ((vox[:, 0] * X + q[:, 0]) * Y + q[:, 1]) * Z + q[:, 2]
        at = np.minimum(np.searchsorted(key, qk), max(len(key) - 1, 0))
        hit = inside & (len(key) > 0) & (key[at] == qk)
        nbr[hit, o] = at[hit]
    pairs = [(np.nonzero(nbr[:, o] >= 0)[0], nbr[nbr[:, o] >= 0, o]) for o in range(K)]
    return dict(valid=valid, slot=slot, rep=rep, voxels=vox, nbr=nbr,
                pairs=pairs, k=k)


def _w(weight, o, k, dtype):
    return np.asarray(weight, dtype)[:, o // (k * k), (o // k) % k, o % k, :]   # [Cout, Cin]


def forward(features, weight, bias, rb, dtype=np.float64):
    x = np.asarray(features, dtype)
    k, M = rb["k"], len(rb["rep"])
    cout = weight.shape[0]
    acc = np.zeros((M, cout), dtype)
    if bias is not None:
        acc += np.asarray(bias, dtype)
    for o, (dst, src) in enumerate(rb["pairs"]):
        acc[dst] += x[rb["rep"][src]] @ _w(weight, o, k, dtype).T
    out = np.zeros((x.shape[0], cout), dtype)
    out[rb["valid"]] = acc[rb["slot"][rb["valid"]]]
    return out


def backward(features, weight, grad_out, rb, dtype=np.float64):
    """(grad_features, grad_weight, grad_bias)"""
    x = np.asarray(features, dtype)
    g = np.asarray(grad_out, dtype)
    k, M = rb["k"], len(rb["rep"])
    dysum = np.zeros((M, g.shape[1]), dtype)
    np.add.at(dysum, rb["slot"][rb["valid"]], g[rb["valid"]])
    dx_slot = np.zeros((M, x.shape[1]), dtype)
    gw = np.zeros(weight.shape, dtype)
    for o, (dst, src) in enumerate(rb["pairs"]):
        np.add.at(dx_slot, src, dysum[dst] @ _w(weight, o, k, dtype))
        gw[:, o // (k * k), (o // k) % k, o % k, :] = dysum[dst].T @ x[rb["rep"][src]]
    gx = np.zeros_like(x)
    gx[rb["rep"]] = dx_slot
    return gx, gw, dysum.sum(0)


def torch_reference(features, weight, bias, grad_out, rb, dtype, device):
    """The same per-offset pair sums as forward / backward above, restated with torch on `device` in `dtype`, for the
    full-size cases: (out, grad_features, grad_weight, grad_bias).  fp32 matmuls run without TF32."""
    import torch
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        t = lambda a: torch.as_tensor(np.asarray(a), device=device)   # noqa: E731
        x, w, g = t(features).to(dtype), t(weight).to(dtype), t(grad_out).to(dtype)
        k, M = rb["k"], len(rb["rep"])
        rep, slot, valid = t(rb["rep"]), t(rb["slot"]), t(rb["valid"])
        acc = torch.zeros(M, w.shape[0], dtype=dtype, device=device)
        if bias is not None:
            acc += t(bias).to(dtype)
        dysum = torch.zeros(M, g.shape[1], dtype=dtype, device=device).index_add_(0, slot[valid], g[valid])
        dx = torch.zeros(M, x.shape[1], dtype=dtype, device=device)
        gw = torch.zeros_like(w)
        for o, (dst, src) in enumerate(rb["pairs"]):
            dst, src = t(dst), t(src)
            wo = w[:, o // (k * k), (o // k) % k, o % k, :]
            xs = x[rep[src]]
            acc.index_add_(0, dst, xs @ wo.T)
            dx.index_add_(0, src, dysum[dst] @ wo)
            gw[:, o // (k * k), (o // k) % k, o % k, :] = dysum[dst].T @ xs
        out = torch.zeros(x.shape[0], w.shape[0], dtype=dtype, device=device)
        out[valid] = acc[slot[valid]]
        gx = torch.zeros_like(x)
        gx[rep] = dx
        return [a.double().cpu().numpy() for a in (out, gx, gw, dysum.sum(0))]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
