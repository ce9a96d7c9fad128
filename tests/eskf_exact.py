"""The filter updates of eskf.cc restated in extended precision, each with a componentwise first-order bound on the error of
the fp64 computation of the same formula, and checks that hold a computed filter against them.

Every function takes the fp64 inputs the device read (state, covariance, rows or measurements) and works on them in mpmath
at DPS digits: no result depends on the order of a summation. The discrete rules of the reference are reproduced exactly:

  the N == 1 rule           A, b scaled by sum R / (sum R + 1e-4)  (eskf.cc:100)
  a zero step               when the count is 0 or the system matrix is exactly singular (the zero pivot of warp_solve6 /
                            warp_gauss_jordan); x and P are then returned unchanged
  the Exp thresholds        1e-5 in so3_exp3 (State (+)), 1e-7 in so3_exp_vec (getFx)
  no symmetrisation         P66 = P[0:6, 0:6] read as given, P - K H P left asymmetric

The error scales follow the form the device computes, not the problem: a sum of d levels costs gamma_d sum|terms|
(gamma_d = d u / (1 - d u), u = 2^-53); a solve propagates Skeel-style,
  |dy| <= |M^-1| (|dM| |y| + |db|) + c u |M^-1| |M| |y|,
and a product picks up the errors of its factors. A check asserts |computed - exact| <= K scale entry by entry, one K per
quantity, and reports the worst ratio and where it was reached (printed, so pytest -s shows them)."""
import math
import os

import mpmath
import numpy as np

DPS = 40
U = 2.0 ** -53
TH_EXP3 = 1e-5   # so3_exp3 (math_utils.hpp:55-68): identity at or below
TH_EXPV = 1e-7   # so3_exp_vec (math_utils.hpp:20-32)
N1_EPS = 1e-4    # eskf.cc:100

# Bounds, in units of each quantity's own scale: powers of two, each at least 4x the worst ratio measured on the device
# (tests/test_gpu_filter_exact.py, an H100 80GB HBM3 at a 700 W power limit) and above the oracle's worst in the same
# units (tests/test_eskf_exact.py, information form).
K_STEP = 4.0     # LiDAR update, |x - x_exact| / (d delta + u |x|) outside the attitude: device 0.82, oracle 0.79
K_POSE = 0.5     # LiDAR update, |Log(R_exact^T R)| / (|d delta_theta| + 8u): device 0.059, oracle 0.12
K_COV = 4.0      # LiDAR update, |P - P_exact| / dP: device 0.92, oracle 0.80
K_OBS = 4.0      # dense inertial / kinematic update, state, attitude and covariance: device 0.89, oracle 0.89.
#                The Skeel form cannot see K = P H^T S^-1 cancel the solve's error: at cond(S) >= 1e6 (m = 15, 18 with
#                kin_meas_noise = 1e-12) the bound is 1e5 - 1e12 times the measured error, so those cases test little
K_PRED = 4.0     # predict, state, attitude and covariance: device 0.67, oracle 0.79


def gamma(d):
    return d * U / (1.0 - d * U)


# ---- summation depth of each device path (the d of gamma_d) ---------------------------------------------------------
def depth_rows(n):
    """k_update_by_points (lk_filter.cu): ceil(n / 256) rows serially per thread, 5 levels of the warp's transposing tree,
    the 8 warps added in order."""
    return math.ceil(n / 256) + 5 + 8


def depth_scan(n):
    """The scan paths and the pose scorer (lk_residual.cu, lk_fused.cu, lk_stream2.cu, lk_score.cu; lk_solve.cuh:
    block_sum_partials and lk_llsync.cuh). One bound for all of them, from the structure they share: a thread's rows
    serially (at most ceil(n / 256): every point of the bucket in one chunk row of a 256-thread block), the warp's tree
    (5), the block's 8 warps, the LK_GROUP = 8 chunk rows of a group, then one group row per LK_GROUP chunks of at least
    128 points. Each path's own depth is smaller (the batch-of-one kernel holds at most one 256-point chunk per block; the
    throughput family's 3 840-point chunks give fewer groups), so the bound is loose by at most the ratio of the first
    term to the real per-thread count."""
    return math.ceil(n / 256) + 5 + 8 + 8 + math.ceil(math.ceil(n / 128) / 8)


# ---- mpmath <-> numpy -------------------------------------------------------------------------------------------------
def mp(a):
    a = np.asarray(a, np.float64)
    if a.ndim == 1:
        return mpmath.matrix([mpmath.mpf(float(v)) for v in a])
    return mpmath.matrix([[mpmath.mpf(float(v)) for v in row] for row in a])


def fl(M):
    """An mpmath matrix (or vector) rounded to float64."""
    return np.array([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)]).reshape(
        (M.rows,) if M.cols == 1 else (M.rows, M.cols))


def absdiff(dev, M):
    """|dev - M| entry by entry, the difference taken at DPS digits."""
    dev = np.asarray(dev, np.float64)
    flat = dev.ravel()
    out = np.array([float(abs(mpmath.mpf(float(flat[k])) - M[k // M.cols, k % M.cols] if M.cols > 1 else
                                   mpmath.mpf(float(flat[k])) - M[k]))
                    for k in range(flat.size)])
    return out.reshape(dev.shape)


def _eye(n):
    return mpmath.eye(n)


def exp3(v, threshold):
    """Exp(v) (Rodrigues) at DPS digits, the identity at or below `threshold` as the reference's Exp."""
    v = [mpmath.mpf(x) for x in v]
    nrm = mpmath.sqrt(v[0] ** 2 + v[1] ** 2 + v[2] ** 2)
    # an input within 1e-12 of the threshold has no exact branch to compare against: a test must not produce one
    assert not abs(nrm - threshold) <= 1e-12 * threshold, ("step within 1e-12 of the Exp threshold", float(nrm), threshold)
    E = _eye(3)
    if nrm > threshold:
        k = [x / nrm for x in v]
        K = mpmath.matrix([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        E = E + mpmath.sin(nrm) * K + (1 - mpmath.cos(nrm)) * (K * K)
    return E


def att_err(R_dev, R_ex):
    """|Log(R_ex^T R_dev)| to first order: the vee of the skew part of R_ex^T R_dev (its symmetric part is the
    non-orthonormality both carry from their fp64 input)."""
    D = R_ex.T * mp(np.asarray(R_dev, np.float64).reshape(3, 3))
    return float(mpmath.sqrt(((D[2, 1] - D[1, 2]) / 2) ** 2 + ((D[0, 2] - D[2, 0]) / 2) ** 2 + ((D[1, 0] - D[0, 1]) / 2) ** 2))


def _x36(x):
    x = np.asarray(x)
    return np.asarray(x.view(np.float64) if x.dtype.names is None else np.ascontiguousarray(x).view(np.float64),
                      np.float64).reshape(36)


def boxplus(x36, d):
    """State::operator+= (eskf.cc:18-29) at DPS digits: R Exp(d_theta) (threshold 1e-5), the rest added."""
    R = mp(x36[:9].reshape(3, 3)) * exp3([d[0], d[1], d[2]], TH_EXP3)
    rest = [mpmath.mpf(float(x36[9 + i])) + d[3 + i] for i in range(27)]
    return R, rest


# ---- the information-form LiDAR update (eskf.cc:91-113) ---------------------------------------------------------------
def info_sums(h, z, r, dps=DPS):
    """A = s sum h^T h / R (6 x 6), b = s sum h^T z / R, s the N == 1 scale, and the sums of the absolute terms."""
    h = np.asarray(h, np.float64).reshape(-1, 6); z = np.asarray(z, np.float64); r = np.asarray(r, np.float64)
    n = len(z)
    with mpmath.workdps(dps):
        w = [1 / mpmath.mpf(float(v)) for v in r]
        hw = [[mpmath.mpf(float(h[k, a])) * w[k] for a in range(6)] for k in range(n)]
        A = mpmath.matrix(6, 6); b = mpmath.matrix(6, 1)
        for a in range(6):
            for c in range(a, 6):
                A[a, c] = A[c, a] = mpmath.fsum(hw[k][a] * float(h[k, c]) for k in range(n))
            b[a] = mpmath.fsum(hw[k][a] * float(z[k]) for k in range(n))
        s = mpmath.mpf(1)
        if n == 1:
            sr = mpmath.mpf(float(r[0]))
            s = sr / (sr + mpmath.mpf(N1_EPS))
        A = A * s; b = b * s
    ah = np.abs(h) / r[:, None]
    Aabs = float(s) * (ah.T @ np.abs(h)); babs = float(s) * (ah.T @ np.abs(z))
    return A, b, Aabs, babs, n


def update_exact(x, P, h, z, r, depth, dps=DPS):
    """ESKF::updateByPoints in information form on the fp64 inputs, and the error scales of the device's computation of
    the same form with sums of `depth` levels. Returns a dict: x (R 3 x 3 and the other 27 entries, mpmath), P (mpmath
    30 x 30), delta, the scales d_delta [30], d_att, dP [30, 30], the count, whether the step is zero, and cond(M) beside
    the condition number of the problem's own form (the posterior information P66^-1 + A)."""
    x36 = _x36(x)
    Pn = np.asarray(P, np.float64).reshape(30, 30)
    with mpmath.workdps(dps):
        A, b, Aabs, babs, n = info_sums(h, z, r, dps)
        Pm = mp(Pn)
        P66 = Pm[0:6, 0:6]
        M = _eye(6) + A * P66
        zero = n == 0 or mpmath.det(M) == 0
        out = dict(n=n, zero=zero, depth=depth)
        if zero:
            out.update(R=mp(x36[:9].reshape(3, 3)), rest=[mpmath.mpf(float(v)) for v in x36[9:]], P=Pm,
                       delta=mpmath.matrix(30, 1), d_delta=np.zeros(30), d_att=0.0, dP=np.zeros((30, 30)),
                       d_rest=np.zeros(27), cond_M=np.inf, cond_problem=np.nan)
            return out
        Mi = mpmath.inverse(M)
        y = Mi * b
        W = Mi * A
        P6 = Pm[:, 0:6]
        delta = P6 * y
        R, rest = boxplus(x36, delta)
        Pnew = Pm - P6 * (W * Pm[0:6, :])
        yf, Wf, Mf, Mif = fl(y), fl(W), fl(M), fl(Mi)
    Af = fl(A)
    aP = np.abs(Pn); aP66 = aP[:6, :6]; aP6 = aP[:, :6]; aProw = aP[:6, :]
    aMi = np.abs(Mif)
    dA = gamma(depth + 3 + (2 if n == 1 else 0)) * Aabs
    db = gamma(depth + 3 + (2 if n == 1 else 0)) * babs
    dM = dA @ aP66 + gamma(7) * np.abs(Af) @ aP66
    dy = aMi @ (dM @ np.abs(yf) + db) + 6 * U * aMi @ np.abs(Mf) @ np.abs(yf)
    dW = aMi @ (dM @ np.abs(Wf) + dA) + 6 * U * aMi @ np.abs(Mf) @ np.abs(Wf)
    d_delta = aP6 @ dy + gamma(6) * aP6 @ np.abs(yf)
    dP = U * (aP + 7 * aP6 @ np.abs(Wf) @ aProw) + aP6 @ dW @ aProw
    rest_f = np.array([float(v) for v in rest])
    out.update(R=R, rest=rest, P=Pnew, delta=delta, d_delta=d_delta, d_att=float(d_delta[:3].sum()) + 8 * U,
               d_rest=d_delta[3:] + U * np.abs(rest_f), dP=dP, cond_M=float(np.linalg.cond(Mf)),
               cond_problem=_cond_problem(h, r, Pn))
    return out


def _cond_problem(h, r, P):
    """cond of the posterior information matrix P66^-1 + A (the problem's own conditioning, whatever n), nan when P66 is
    singular."""
    h = np.asarray(h, np.float64).reshape(-1, 6)
    P66 = np.asarray(P, np.float64).reshape(30, 30)[:6, :6]
    if len(h) == 0 or np.linalg.matrix_rank(P66) < 6:
        return np.nan
    A = (h / np.asarray(r, np.float64)[:, None]).T @ h
    return float(np.linalg.cond(np.linalg.inv(P66) + A))


# ---- the dense inertial / kinematic update (eskf.cc:125-145) ----------------------------------------------------------
def dense_exact(x, P, H, z, r, dH=None, dz=None, dps=DPS):
    """K = P H^T S^-1, S = H P H^T + diag(r), x (+)= K z, P -= K H P on fp64 (or mpmath) H, z; dH, dz are the errors the
    computed H and z carry (0 when they are exact)."""
    x36 = _x36(x)
    Pn = np.asarray(P, np.float64).reshape(30, 30)
    with mpmath.workdps(dps):
        Hm = H if isinstance(H, mpmath.matrix) else mp(H)
        zm = z if isinstance(z, mpmath.matrix) else mp(z)
        m = Hm.rows
        Pm = mp(Pn)
        PHT = Pm * Hm.T
        S = Hm * PHT
        for a in range(m):
            S[a, a] += mpmath.mpf(float(r[a]))
        HP = Hm * Pm
        out = dict(m=m)
        if mpmath.det(S) == 0:
            out.update(zero=True, R=mp(x36[:9].reshape(3, 3)), rest=[mpmath.mpf(float(v)) for v in x36[9:]], P=Pm,
                       d_att=0.0, d_rest=np.zeros(27), dP=np.zeros((30, 30)), cond_S=np.inf)
            return out
        Si = mpmath.inverse(S)
        Xz = Si * zm
        XHP = Si * HP
        delta = PHT * Xz
        R, rest = boxplus(x36, delta)
        Pnew = Pm - PHT * XHP
        Hf, PHTf, Sf, Sif, Xzf, XHPf = fl(Hm), fl(PHT), fl(S), fl(Si), fl(Xz), fl(XHP)
    Xzf = Xzf.reshape(m); Hf = Hf.reshape(m, 30); PHTf = PHTf.reshape(30, m)
    dH = np.zeros((m, 30)) if dH is None else dH
    dz = np.zeros(m) if dz is None else dz
    aP, aH, aPHT, aSi = np.abs(Pn), np.abs(Hf), np.abs(PHTf), np.abs(Sif)
    dPHT = gamma(30) * aP @ aH.T + aP @ dH.T
    dHP = gamma(30) * aH @ aP + dH @ aP
    dS = gamma(31) * aH @ aPHT + aH @ dPHT + dH @ aPHT + U * np.abs(np.diag(np.asarray(r, np.float64)))
    dXz = aSi @ (dS @ np.abs(Xzf) + dz) + m * U * aSi @ np.abs(Sf) @ np.abs(Xzf)
    dXHP = aSi @ (dS @ np.abs(XHPf) + dHP) + m * U * aSi @ np.abs(Sf) @ np.abs(XHPf)
    d_delta = aPHT @ dXz + dPHT @ np.abs(Xzf) + gamma(m) * aPHT @ np.abs(Xzf)
    dP = U * aP + aPHT @ dXHP + dPHT @ np.abs(XHPf) + gamma(m) * aPHT @ np.abs(XHPf)
    rest_f = np.array([float(v) for v in rest])
    out.update(zero=False, R=R, rest=rest, P=Pnew, d_att=float(d_delta[:3].sum()) + 8 * U,
               d_rest=d_delta[3:] + U * np.abs(rest_f), dP=dP, cond_S=float(np.linalg.cond(Sf)))
    return out


def _skew(v):
    return mpmath.matrix([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def _skew_abs(v):
    v = np.abs(np.asarray(v, np.float64))
    return np.array([[0, v[2], v[1]], [v[2], 0, v[0]], [v[1], v[0], 0]])


def obs_rows(x, meas, cfg, gravity, acc_norm, kin):
    """H (m x 30), z, r of KILO::predictUpdateImu / predictUpdateKinImu's observation (KILO.cc:243-310) at DPS digits from
    the fp64 state and sample, with the errors dH, dz of their fp64 computation."""
    x36 = _x36(x)
    legs = [i for i in range(4) if kin and int(meas["contact"][i]) != 0]
    m = 6 + 3 * len(legs)
    H = mpmath.matrix(m, 30); z = mpmath.matrix(m, 1)
    dH = np.zeros((m, 30)); dz = np.zeros(m)
    r = np.zeros(m)
    sc = mpmath.mpf(float(gravity)) / mpmath.mpf(float(acc_norm))
    scf = float(gravity) / float(acc_norm)
    for a in range(6):
        H[a, 9 + a] = 1; H[a, 18 + a] = 1
        if a < 3:
            z[a] = sc * float(meas["acc"][a]) - float(x36[24 + a]) - float(x36[15 + a])
            dz[a] = gamma(3) * (abs(scf * float(meas["acc"][a])) + abs(x36[24 + a]) + abs(x36[15 + a])) + \
                gamma(2) * abs(scf * float(meas["acc"][a]))
        else:
            z[a] = mpmath.mpf(float(meas["gyr"][a - 3])) - float(x36[27 + a - 3]) - float(x36[18 + a - 3])
            dz[a] = gamma(2) * (abs(float(meas["gyr"][a - 3])) + abs(x36[24 + a]) + abs(x36[15 + a]))
        r[a] = cfg["imu_acc_meas_noise"] if a < 2 else (cfg["imu_acc_z_meas_noise"] if a == 2 else cfg["imu_gyr_meas_noise"])
    Rm = mp(x36[:9].reshape(3, 3)); aR = np.abs(x36[:9].reshape(3, 3))
    w = [mpmath.mpf(float(v)) for v in x36[27:30]]; wf = x36[27:30]
    for c, leg in enumerate(legs):
        fp = [mpmath.mpf(float(v)) for v in meas["foot_pos"][leg]]; fpf = np.asarray(meas["foot_pos"][leg], np.float64)
        fv = [mpmath.mpf(float(v)) for v in meas["foot_vel"][leg]]; fvf = np.asarray(meas["foot_vel"][leg], np.float64)
        u = [w[1] * fp[2] - w[2] * fp[1] + fv[0], w[2] * fp[0] - w[0] * fp[2] + fv[1], w[0] * fp[1] - w[1] * fp[0] + fv[2]]
        ua = np.array([abs(wf[1] * fpf[2]) + abs(wf[2] * fpf[1]), abs(wf[2] * fpf[0]) + abs(wf[0] * fpf[2]),
                       abs(wf[0] * fpf[1]) + abs(wf[1] * fpf[0])]) + np.abs(fvf)
        Hth = -(Rm * _skew(u)); Hw = -(Rm * _skew(fp))
        dHth = gamma(3) * aR @ _skew_abs(ua) + aR @ _skew_abs(gamma(2) * ua)
        dHw = gamma(3) * aR @ _skew_abs(fpf)
        Ru = Rm * mpmath.matrix(u)
        for q in range(3):
            row = 6 + 3 * c + q
            for k in range(3):
                H[row, k] = Hth[q, k]; H[row, 21 + k] = Hw[q, k]
                dH[row, k] = dHth[q, k]; dH[row, 21 + k] = dHw[q, k]
            H[row, 6 + q] = 1
            z[row] = -mpmath.mpf(float(x36[12 + q])) - Ru[q]
            dz[row] = gamma(4) * (abs(x36[12 + q]) + aR[q] @ ua) + aR[q] @ (gamma(2) * ua)
            r[row] = cfg["kin_meas_noise"]
    return H, z, r, dH, dz


# ---- the predict (eskf.cc:64-89) --------------------------------------------------------------------------------------
def predict_exact(x, P, Q, dt, prop_state=True, prop_cov=True, dps=DPS):
    """ESKF::predict as k_predict_dt runs it: the state first (getFunctionf, State (+)), then F P F^T + dt^2 Q with F from
    the updated state (getFx, Exp threshold 1e-7)."""
    x36 = _x36(x).copy()
    Pn = np.asarray(P, np.float64).reshape(30, 30); Qn = np.asarray(Q, np.float64).reshape(30, 30)
    out = dict(dt=dt)
    with mpmath.workdps(dps):
        dtm = mpmath.mpf(float(dt))
        Rm = mp(x36[:9].reshape(3, 3))
        R, rest = Rm, [mpmath.mpf(float(v)) for v in x36[9:]]
        d_att, d_rest = 0.0, np.zeros(27)
        aR = np.abs(x36[:9].reshape(3, 3))
        if prop_state:
            a = mp(x36[24:27]); g = mp(x36[21:24])
            Ra = Rm * a
            d = [dtm * float(x36[27 + k]) for k in range(3)] + [dtm * float(x36[12 + k]) for k in range(3)] + \
                [dtm * (Ra[k] + g[k]) for k in range(3)] + [0] * 21
            R, rest = boxplus(x36, d)
            dd = np.zeros(30)
            dd[:3] = U * np.abs(dt * x36[27:30]); dd[3:6] = U * np.abs(dt * x36[12:15])
            dd[6:9] = gamma(5) * abs(dt) * (aR @ np.abs(x36[24:27]) + np.abs(x36[21:24]))
            rest_f = np.array([float(v) for v in rest])
            d_att = float(dd[:3].sum()) + 8 * U
            d_rest = dd[3:] + U * np.abs(rest_f)
        out.update(R=R, rest=rest, d_att=d_att, d_rest=d_rest)
        Pm = mp(Pn)
        if not prop_cov:
            out.update(P=Pm, dP=np.zeros((30, 30)))
            return out
        # F from the updated state: R after the state step, imu_a and imu_w unchanged by it
        Rs = R
        w = x36[27:30]; a = x36[24:27]
        F = _eye(30)
        E = exp3([-dtm * float(w[0]), -dtm * float(w[1]), -dtm * float(w[2])], TH_EXPV)
        RK = -dtm * (Rs * _skew([mpmath.mpf(float(v)) for v in a]))
        for i in range(3):
            for j in range(3):
                F[i, j] = E[i, j]
                F[6 + i, j] = RK[i, j]
                F[6 + i, 18 + j] = dtm * Rs[i, j]
            F[i, 21 + i] = dtm
            F[3 + i, 6 + i] = dtm
            F[6 + i, 15 + i] = dtm
        Pnew = F * Pm * F.T + (dtm * dtm) * mp(Qn)
        Ff = fl(F)
    aF = np.abs(Ff)
    # the fp64 F: Exp (a few u absolute), -dt R [a]x (3-term products of a rounded R), dt R
    dF = np.zeros((30, 30))
    dF[:3, :3] = 4 * U
    dF[6:9, :3] = gamma(5) * abs(dt) * aR @ _skew_abs(a)
    dF[6:9, 18:21] = gamma(2) * abs(dt) * aR
    aP = np.abs(Pn)
    dP = gamma(10) * (aF @ aP @ aF.T) + dF @ aP @ aF.T + aF @ aP @ dF.T + gamma(3) * dt * dt * np.abs(Qn)
    out.update(P=Pnew, dP=dP)
    return out


# ---- checks -----------------------------------------------------------------------------------------------------------
def _ratio(err, scale):
    err = np.asarray(err, np.float64); scale = np.asarray(scale, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(err == 0, 0.0, err / scale)
    return q


def check(x_dev, P_dev, ex, k_state, k_att, k_cov, what="", bitwise_if_zero=True, x_in=None, P_in=None):
    """Asserts the computed filter (x_dev, P_dev) against an exact result of update_exact / dense_exact /
    predict_exact: every non-attitude state entry, the attitude as |Log(R_exact^T R)|, every covariance entry, each
    within its K times its scale. A zero step must return x_in / P_in bit for bit. Returns (state, attitude, cov) ratios."""
    x36 = _x36(x_dev)
    Pd = np.asarray(P_dev, np.float64).reshape(30, 30)
    test = os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0]
    if ex.get("zero") and bitwise_if_zero and x_in is not None:
        assert x36.tobytes() == _x36(x_in).tobytes(), (what, "zero step moved x")
        assert Pd.tobytes() == np.asarray(P_in, np.float64).reshape(30, 30).tobytes(), (what, "zero step moved P")
        print(f"eskf-exact {test} {what}: zero step, x and P returned bit for bit")
        return 0.0, 0.0, 0.0
    with mpmath.workdps(DPS):
        e_rest = np.array([float(abs(mpmath.mpf(float(x36[9 + i])) - ex["rest"][i])) for i in range(27)])
        e_att = att_err(x36[:9], ex["R"])
        e_P = absdiff(Pd, ex["P"])
    q_state = _ratio(e_rest, ex["d_rest"])
    q_att = 0.0 if e_att == 0 else (e_att / ex["d_att"] if ex["d_att"] > 0 else np.inf)
    q_cov = _ratio(e_P, ex["dP"])
    ks = int(np.argmax(q_state)); kc = np.unravel_index(int(np.argmax(q_cov)), q_cov.shape)
    rs, rc = float(q_state[ks]), float(q_cov[kc])
    dg = np.abs(np.diag(fl(ex["P"])))
    corr = e_P / np.sqrt(np.maximum(np.outer(dg, dg), 1e-300))
    cond = f"cond(M) {ex['cond_M']:.2g} cond(P66^-1+A) {ex['cond_problem']:.2g}" if "cond_M" in ex else (
        f"cond(S) {ex['cond_S']:.2g}" if "cond_S" in ex else "")
    if P_in is not None:  # what P - K H P cancels: prior over posterior variance, the covariance form's own conditioning
        d_in = np.abs(np.diag(np.asarray(P_in, np.float64).reshape(30, 30)))
        cond += f" cancellation {float(np.max(d_in / np.maximum(dg, 1e-300))):.2g}"
    print(f"eskf-exact {test} {what}: worst/scale state {rs:.3g} at x[{9 + ks}] attitude {q_att:.3g} cov {rc:.3g} at "
          f"P{tuple(int(v) for v in kc)} | cov err {float(corr.max()):.3g} corr units | {cond}")
    assert rs <= k_state, (what, "state", rs, int(9 + ks), e_rest[ks], ex["d_rest"][ks])
    assert q_att <= k_att, (what, "attitude", q_att, e_att, ex["d_att"])
    assert rc <= k_cov, (what, "cov", rc, tuple(int(v) for v in kc), e_P[kc], ex["dP"][kc])
    return rs, q_att, rc


# ---- scenarios shared by the CPU and the device tests -----------------------------------------------------------------
GEOMETRIES = ("box", "plane", "corridor", "far")
PRIORS = ("init", "dense", "asym", "wide", "scaled", "corr", "zero_theta", "pivot")


def rows(geometry, n, g):
    """n LiDAR-like rows h = [p x n_w, n_w] (the sign and frame of lk_point.cuh's row do not matter to the algebra): the
    box room (six wall normals), one plane (rank-3 A), a corridor of two parallel walls and a floor (rank 5), or the box
    room 1 km from the origin (theta columns ~1e3)."""
    if geometry == "plane":
        nrm = np.tile([0.0, 0.0, 1.0], (n, 1))
    elif geometry == "corridor":
        nrm = np.array([[0.0, 1.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, 1.0]])[g.integers(0, 3, n)]
    else:
        nrm = np.vstack([np.eye(3), -np.eye(3)])[g.integers(0, 6, n)]
        nrm = nrm + 0.05 * g.standard_normal((n, 3))
        nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    p = g.uniform(-4.0, 4.0, (n, 3))
    if geometry == "far":
        p += (700.0, -650.0, 300.0)
    return np.hstack([np.cross(p, nrm), nrm])


def weights(kind, n, g):
    if kind == "wide":
        return 10.0 ** g.uniform(-8.0, 2.0, n)
    if kind == "tiny":
        return np.full(n, 1e-8)
    return g.uniform(1e-3, 1e-2, n)


def prior(kind, g, h=None, r=None):
    """A 30 x 30 prior: init_cov, dense_cov, dense_cov skewed (asymmetric), theta and p sd 10 (A P66 ~ 1e10 against
    R = 1e-8), theta sd 1e-6 against p sd 10, theta-p correlation 1 - 1e-9, a zero theta block, or (needs the rows) a P66
    for which I + A P66 has a leading pivot ~1e-16 of its largest entry, so that the solve must swap rows."""
    import general_prior as gp
    if kind == "init":
        return 1e-6 * np.eye(30)
    P = gp.dense_cov(g).reshape(30, 30)
    if kind == "dense":
        return P
    if kind == "asym":
        return np.asarray(gp.skewed(P, g, rel=1e-6)).reshape(30, 30)
    if kind == "zero_theta":
        P = P.copy(); P[:3, :] = 0.0; P[:, :3] = 0.0
        return P
    sd = np.sqrt(np.diag(P))
    C = P / np.outer(sd, sd)
    if kind == "wide":
        sd[:6] = 10.0
    elif kind == "scaled":
        sd[:3] = 1e-6; sd[3:6] = 10.0
    elif kind == "corr":
        sd[:6] = (2e-3, 3e-3, 4e-3, 2e-3, 3e-3, 4e-3)
        C[:6, :] = 0.0; C[:, :6] = 0.0
        C[:6, :6] = np.kron(np.array([[1.0, 1 - 1e-9], [1 - 1e-9, 1.0]]), np.eye(3))
    elif kind == "pivot":
        A = (h / r[:, None]).T @ h
        Mt = np.eye(6)[[1, 0, 2, 3, 4, 5]] + 0.5 * np.eye(6)[[0, 1, 3, 2, 5, 4]]
        Mt[0, 0] = 0.0
        Pp = P.copy()
        Pp[:6, :6] = np.linalg.solve(A, Mt - np.eye(6))
        return Pp
    P = C * np.outer(sd, sd)
    return P


def state(g, far=False):
    import general_prior as gp
    return gp.prior_at(gp.so3_uniform(g), (800.0, -650.0, 30.0) if far else (12.0, -7.5, 0.4), g)


def observe(h, r, step, g):
    """z = h step + noise of variance R: a measurement that pulls the state by about `step` (6) when the prior is wide."""
    return h @ np.asarray(step, np.float64) + np.sqrt(r) * g.standard_normal(len(r))


SCENARIOS = [  # (geometry, n, weights, prior, step)
    ("box", 1, "fixed", "dense", None), ("box", 2, "fixed", "init", None), ("box", 5, "wide", "dense", None),
    ("box", 6, "fixed", "asym", None), ("box", 255, "wide", "dense", None), ("box", 257, "fixed", "init", None),
    ("plane", 300, "fixed", "dense", None), ("corridor", 300, "wide", "dense", None), ("far", 300, "fixed", "dense", None),
    ("box", 300, "tiny", "wide", (1.0, -0.2, 0.3, 1.0, 2.0, -1.0)), ("box", 300, "tiny", "wide", (2.0, -2.0, 1.0, 0, 0, 0)),
    ("box", 300, "fixed", "scaled", None), ("box", 300, "fixed", "corr", None), ("box", 300, "fixed", "zero_theta", None),
    ("box", 6, "fixed", "pivot", None), ("box", 3000, "wide", "dense", None),
]


def scenario_id(s):
    return f"{s[0]}-{s[1]}-{s[2]}-{s[3]}" + ("-step" if s[4] else "")


def case(geometry, n, weight, prior_kind, seed, step=(0.0,) * 6):
    """(x, P [900], h, z, r) of one scenario."""
    from legkilo_b200 import synth
    g = synth.rng(seed)
    h = rows(geometry, n, g)
    r = weights(weight, n, g)
    P = prior(prior_kind, g, h, r)
    x = state(g, far=geometry == "far")
    z = observe(h, r, step, g)
    return x, P.ravel(), h, z, r


def record_exact(h, z, r, dps=DPS):
    """The lk_score_poses record of rows (include/legkilo_b200.h: LK_SCORE_*): A's upper triangle, b, sum R, the count
    and sum z^2 / R, each summed exactly; and per entry the sum of the absolute values of its terms."""
    h = np.asarray(h, np.float64).reshape(-1, 6); z = np.asarray(z, np.float64); r = np.asarray(r, np.float64)
    iu = np.triu_indices(6)
    with mpmath.workdps(dps):
        w = [1 / mpmath.mpf(float(v)) for v in r]
        hw = [[mpmath.mpf(float(h[k, a])) * w[k] for a in range(6)] for k in range(len(z))]
        rec = [mpmath.fsum(hw[k][a] * float(h[k, c]) for k in range(len(z))) for a, c in zip(*iu)]
        rec += [mpmath.fsum(hw[k][a] * float(z[k]) for k in range(len(z))) for a in range(6)]
        rec += [mpmath.fsum(mpmath.mpf(float(v)) for v in r), mpmath.mpf(len(z)),
                mpmath.fsum(mpmath.mpf(float(q)) ** 2 * w[k] for k, q in enumerate(z))]
    ah = np.abs(h) / r[:, None]
    scale = np.concatenate([(ah.T @ np.abs(h))[iu], ah.T @ np.abs(z), [np.abs(r).sum(), 0.0, float((z * z / r).sum())]])
    return rec, scale
