"""init_plane (voxel_map.cc:42-117) restated in extended precision, and a walker that holds every plane fit a map blob
keeps against it.

The reference forms the covariance with the one-pass formula  sum p p^T / N - c c^T,  so its rounding error grows with
S = max_i |p_i|^2 (the moments) and the normal's error with S over the eigen-gap  gap = l_mid - l_min.  No fixed
tolerance fits both a voxel at the origin and one 10 km out, so every bound below is scaled to the plane's own
conditioning:

  centre     K_c eps max|p|           normal     K_n eps S / gap
  plane_var  K_v eps S / gap, relative to its largest entry
  d, radius  one float ulp of the exact value plus the centre and normal errors it inherits
  is_plane   exact whenever the exact l_min lies outside  threshold +- K_b eps S

Here the centre and the covariance are exact: the float64 points are scaled to integers and the moments summed in
Python integers, then rounded once to DPS digits. The eigen step runs in mpmath at DPS digits, plane_var in
np.longdouble. None of it depends on the order of a summation."""
import os

import mpmath
import numpy as np

from legkilo_b200 import abi

EPS = float(np.finfo(np.float64).eps)
DPS = 40
LD = np.longdouble


def _as_ints(pw):
    """The points as integers over one power-of-two denominator: pw = ints / den exactly."""
    vals = [float(v) for v in np.asarray(pw, np.float64).ravel()]
    ratios = [v.as_integer_ratio() for v in vals]
    den = max(d for _, d in ratios)
    ints = [n * (den // d) for n, d in ratios]
    return [ints[3 * i:3 * i + 3] for i in range(len(vals) // 3)], den


def _var6(var):
    """[n, 6] upper triangles (xx xy xz yy yz zz) -> [n, 3, 3]."""
    v = np.asarray(var, np.float64).reshape(-1, 6)
    return v[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)


def init_plane_exact(pw, var, planer_threshold, dps=DPS):
    """init_plane of float64 points pw [n, 3] with covariances var ([n, 6] upper triangles or [n, 3, 3]), the threshold a
    float as the reference holds it. Returns the exact fit, the normal sign-canonical (largest |component| positive):
    center, normal (np.longdouble), lam (l_min, l_mid, l_max), radius, d, plane_var (6 x 6, np.longdouble; computed when
    the exact decision is a plane and gap > 0), is_plane, and the conditioning S, rmax = max|p|, gap."""
    pw = np.asarray(pw, np.float64).reshape(-1, 3)
    n = len(pw)
    assert n > 0
    thr = float(np.float32(planer_threshold))  # planer_threshold_ is a float (voxel_map.h)
    with mpmath.workdps(dps):
        P, den = _as_ints(pw)
        s = [sum(p[i] for p in P) for i in range(3)]
        ss = [[sum(p[i] * p[j] for p in P) for j in range(3)] for i in range(3)]
        # centre s / (n den); covariance (n ss - s s^T) / (n den)^2: exact rationals, rounded once here
        c = [mpmath.mpf(s[i]) / (n * den) for i in range(3)]
        nd2 = (n * den) ** 2
        C = mpmath.matrix(3, 3)
        for i in range(3):
            for j in range(3):
                C[i, j] = mpmath.mpf(n * ss[i][j] - s[i] * s[j]) / nd2
        E, Q = mpmath.eigsy(C)
        order = sorted(range(3), key=lambda k: E[k])
        lam = [E[k] for k in order]
        vecs = [[Q[r, k] for r in range(3)] for k in order]  # ascending: e_min, e_mid, e_max
        k = max(range(3), key=lambda r: abs(vecs[0][r]))
        if vecs[0][k] < 0:
            vecs[0] = [-v for v in vecs[0]]
        is_plane = bool(lam[0] < thr)
        gap = lam[1] - lam[0]
        out = dict(n=n, center=np.array([LD(mpmath.nstr(v, dps)) for v in c]),
                   normal=np.array([LD(mpmath.nstr(v, dps)) for v in vecs[0]]),
                   lam=tuple(float(v) for v in lam), is_plane=is_plane, threshold=thr,
                   radius=float(mpmath.sqrt(max(lam[2], 0))), d=float(-sum(vecs[0][i] * c[i] for i in range(3))),
                   gap=float(gap), S=float(max(np.einsum("ij,ij->i", pw, pw))), rmax=float(np.abs(pw).max()),
                   plane_var=None)
        if not is_plane or not gap > 0:
            return out
        # plane_var = sum_i J_i var_i J_i^T, J_i = [sum_{m != min} a_m e_m ((d_i.e_m) e_min + (d_i.e_min) e_m)^T ; I / n]
        # with a_m = 1 / (n (l_min - l_m)) and d_i = p_i - c  (voxel_map.cc:74-92); d_i exact, then long double
        a = [LD(mpmath.nstr(1 / (n * (lam[0] - lam[m])), dps)) for m in (1, 2)]
        D = np.array([[LD(mpmath.nstr(mpmath.mpf(n * p[i] - s[i]) / (n * den), dps)) for i in range(3)] for p in P])
    e = np.array([[LD(mpmath.nstr(v, dps)) for v in vec] for vec in vecs])  # rows e_min, e_mid, e_max
    dmin = D @ e[0]
    G = np.zeros((n, 3, 3), LD)
    for am, em in zip(a, e[1:]):
        row = am * ((D @ em)[:, None] * e[0][None, :] + dmin[:, None] * em[None, :])
        G += em[None, :, None] * row[:, None, :]
    J = np.zeros((n, 6, 3), LD)
    J[:, :3] = G
    J[:, 3:] = np.eye(3, dtype=LD) / LD(n)
    V = np.asarray(var, np.float64)
    V = (V if V.ndim == 3 else _var6(V)).astype(LD)
    JV = np.einsum("nij,njk->nik", J, V)
    out["plane_var"] = np.einsum("nik,njk->ij", JV, J)
    return out


def conditioning(fit):
    """(normal scale eps S / gap, decision band half-width per unit K: eps S)."""
    return (EPS * fit["S"] / fit["gap"] if fit["gap"] > 0 else np.inf), EPS * fit["S"]


# ---- the invariant on a map blob ---------------------------------------------------------------------------------------
# Bounds in units of the plane's conditioning (see the module docstring), each set from the worst ratio measured over the
# device's maps (tests/test_gpu_plane_fits.py, on an H100 80GB HBM3 at 700 W) and the oracle's (tests/test_planefit_exact.py)
K_CENTER = 8.0   # |c - c_exact|_max / (eps max|p|): worst measured 1.2 (device), 2.3 (oracle)
K_NORMAL = 8.0   # |n - n_exact|_max / (eps S / gap): worst measured 0.85 (device), 2.4 (oracle)
K_VAR = 32.0     # |V - V_exact|_max / (|V_exact|_max eps S / gap): worst measured 5.3 (device), 11.9 (oracle)
K_LAM = 8.0      # |l - l_exact| / (eps S), seen through the radius sqrt(l_max): worst measured 0.8 (device), 0 (oracle)
K_BAND = 16.0    # is_plane is pinned wherever |l_min - threshold| > K_BAND eps S: no measured leaf fell inside


def _unpack_var(pv21):
    M = np.zeros((6, 6))
    M[np.triu_indices(6)] = pv21
    return M + np.triu(M, 1).T


def _f32_ulp(x):
    return float(np.spacing(np.abs(np.float32(x))))


def leaves(blob):
    """Every node that holds its points and has been fitted: (node index, the fitted prefix of its points). A leaf with
    pts_count = c and new_points = k was last fitted on its first c - k points, since the reference refits before it
    appends and resets new_points_ at each fit (voxel_map.cc:185-206)."""
    _, roots, nodes, aux, pts = abi.parse_map_blob(blob)
    out = []
    stack = [int(r["node"]) for r in roots]
    while stack:
        i = stack.pop()
        f = int(nodes[i]["flags"])
        mask = (f >> abi.NODE_CHILDMASK_SHIFT) & 0xff
        for ch in range(8):
            if mask & (1 << ch):
                stack.append(int(nodes[i]["child_base"]) + ch)
        c, k = int(aux[i]["pts_count"]), int(aux[i]["new_points"])
        if mask or not (f & abi.NODE_INIT_OCTO) or c - k <= 0:
            continue
        b = int(aux[i]["pts_base"])
        out.append((i, pts[b:b + c - k]))
    return nodes, out


def check_map(blob, cfg, sample=None, seed=0, what=""):
    """Holds every fitted leaf of `blob` (or a seeded sample of `sample` of them) against
    init_plane_exact. Asserts the invariant and returns the worst ratios and counts (printed, so pytest -s shows them)."""
    nodes, lv = leaves(blob)
    thr = cfg["min_eigen_value"]
    max_layer = cfg["max_layer"]
    if sample is not None and len(lv) > sample:
        keep = set(np.random.default_rng(seed).choice(len(lv), sample, replace=False).tolist())
        lv = [x for j, x in enumerate(lv) if j in keep]
    st = dict(leaves=len(lv), planes=0, non_planes=0, in_band=0, max_layer_non_planes=0, center=0.0, normal=0.0,
              var=0.0, d=0.0, radius=0.0, layers=set())
    for i, p in lv:
        A = nodes[i]
        f = int(A["flags"])
        ex = init_plane_exact(p["pw"], p["var"], thr)
        scale, unit = conditioning(ex)
        dist = abs(ex["lam"][0] - ex["threshold"])
        msg = (what, "node", i, "n", ex["n"], "lam", ex["lam"], "threshold", ex["threshold"])
        dev_plane = bool(f & abi.NODE_IS_PLANE)
        st["layers"].add((f >> abi.NODE_LAYER_SHIFT) & 0xff)
        if dist <= K_BAND * unit:
            st["in_band"] += 1
        else:
            assert dev_plane == ex["is_plane"], msg + ("is_plane", dev_plane)
        if not dev_plane:
            st["non_planes"] += 1
            if ((f >> abi.NODE_LAYER_SHIFT) & 0xff) >= max_layer:
                st["max_layer_non_planes"] += 1
            assert ex["lam"][0] >= ex["threshold"] - K_BAND * unit, msg
            continue
        st["planes"] += 1
        assert ex["lam"][0] < ex["threshold"] + K_BAND * unit, msg
        rc = float(np.abs(A["center"].astype(LD) - ex["center"]).max()) / (EPS * ex["rmax"])
        st["center"] = max(st["center"], rc)
        assert rc <= K_CENTER, msg + ("center", rc)
        if not np.isfinite(scale):
            continue
        n = A["normal"].astype(LD)
        flip = float(n @ ex["normal"]) < 0
        if flip:
            n = -n
        rn = float(np.abs(n - ex["normal"]).max()) / scale
        st["normal"] = max(st["normal"], rn)
        assert rn <= K_NORMAL, msg + ("normal", rn, scale)
        V = _unpack_var(A["plane_var"]).astype(LD)
        if flip:
            V[:3, 3:] *= -1; V[3:, :3] *= -1
        Vx = ex["plane_var"]
        rv = float(np.abs(V - Vx).max() / np.abs(Vx).max()) / scale
        st["var"] = max(st["var"], rv)
        assert rv <= K_VAR, msg + ("plane_var", rv, scale)
        # d and radius are floats: the float rounding of the exact value, one ulp either way, plus what they inherit
        d = -float(A["d"]) if flip else float(A["d"])
        nb = K_NORMAL * scale * float(np.abs(ex["center"]).sum()) + K_CENTER * EPS * ex["rmax"]
        rd = (abs(d - float(np.float32(ex["d"]))) - _f32_ulp(ex["d"])) / max(nb, 1e-300)
        st["d"] = max(st["d"], rd)
        assert rd <= 1.0, msg + ("d", d, ex["d"], nb)
        rb = K_LAM * EPS * ex["S"] / (2 * max(ex["radius"], 1e-300))  # |d sqrt(l)| = |d l| / (2 sqrt(l))
        rr = (abs(float(A["radius"]) - float(np.float32(ex["radius"]))) - _f32_ulp(ex["radius"])) / rb
        st["radius"] = max(st["radius"], rr)
        assert rr <= 1.0, msg + ("radius", float(A["radius"]), ex["radius"])
    test = os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0]
    print(f"plane-fit {test} {what}: leaves {st['leaves']} planes {st['planes']} non-planes {st['non_planes']} "
          f"(max layer {st['max_layer_non_planes']}) in-band {st['in_band']} | worst/eps-scale: center {st['center']:.3g} "
          f"normal {st['normal']:.3g} plane_var {st['var']:.3g} d {st['d']:.3g} radius {st['radius']:.3g}")
    return st
