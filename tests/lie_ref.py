"""TEST INFRASTRUCTURE -- extended-precision reference of the Lie layer the kernels use (mink_b200/csrc/bik_math.h).

Every function evaluates its closed form in mpmath at DPS significant digits (more where the closed form cancels) and
rounds the result to fp64, so it is accurate to the last bit of a double at every angle -- unlike the C oracle's fp64 Lie
coefficients, whose closed form for the SO(3) inverse left Jacobian loses ~2 eps / theta^2 below theta ~ 1e-2 (see
tests/test_lie_range_cpu.py::test_oracle_small_angle_band).  The task errors and Jacobians are built from the oracle's
fp64 FK poses and body Jacobians, which are accurate to ~1e-15; only the Lie layer is recomputed here.

Conventions are the kernels': quaternions (w, x, y, z), poses (w, x, y, z, px, py, pz), twists (v, w), and the reference's
identity branch of the SE(3) inverse left Jacobian (Ji = I, Mi = 0 when |w|^2 < 1e-10, mink/lie/se3.py:212-214).
"""

import mpmath as mp
import numpy as np

DPS = 34
IDENTITY_T2 = 1e-10


def _mpf(a):
    return [mp.mpf(float(x)) for x in np.asarray(a, np.float64).ravel()]


def _t2_dps(t2):
    """Digits that keep DPS of them through the (1 - x) / theta^k cancellation at theta^2 = t2."""
    return DPS + (int(-mp.log10(t2)) if 0 < t2 < 1 else 0) * 2 + 10


def _coefs_mp(t2):
    """(A, B, C, D) at theta^2 = t2 (an mpf), at the current precision."""
    if t2 == 0:
        return mp.mpf(1) / 12, mp.mpf(1) / 6, -mp.mpf(1) / 24, mp.mpf(1) / 120
    with mp.workdps(_t2_dps(t2)):
        th = mp.sqrt(t2)
        s, c = mp.sin(th), mp.cos(th)
        A = (1 - th / 2 * mp.cot(th / 2)) / t2
        B = (th - s) / (t2 * th)
        C = (1 - t2 / 2 - c) / (t2 * t2)
        D = (2 * th - 3 * s + th * c) / (2 * t2 * t2 * th)
        return +A, +B, +C, +D


def coefs(t2):
    """coef_A, coef_BCD: [..., 4] = (A, B, C, D) at theta^2 = t2 (fp64 inputs taken as exact)."""
    t2 = np.asarray(t2, np.float64)
    out = np.zeros(t2.shape + (4,))
    with mp.workdps(DPS):
        for i, x in enumerate(t2.ravel()):
            out.reshape(-1, 4)[i] = [float(v) for v in _coefs_mp(mp.mpf(float(x)))]
    return out


# ---- scalar mp building blocks --------------------------------------------------------------------------------------------
def _qmul(a, b):
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]]


def _qconj(a):
    return [a[0], -a[1], -a[2], -a[3]]


def _qnormalize(a):
    n = mp.sqrt(sum(x * x for x in a))
    return [x / n for x in a]


def _qrot(q, v):
    r = _qmul(_qmul(q, [mp.mpf(0)] + list(v)), _qconj(q))
    return r[1:]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _so3_log(q):
    """Rotation vector of the (not necessarily unit) quaternion q, angle in [0, pi] taken on q's w >= 0 hemisphere."""
    n = mp.sqrt(q[1] ** 2 + q[2] ** 2 + q[3] ** 2)
    if n == 0:
        return [mp.mpf(0)] * 3
    sgn = -1 if q[0] < 0 else 1
    f = sgn * 2 * mp.atan2(n, abs(q[0])) / n
    return [f * x for x in q[1:]]


def _se3_log(q, t, w_like=None):
    """(v, w) = log of the pose (q, t).  w_like: at theta = pi, where w and -w are both logs, take the one on its side."""
    w = _so3_log(q)
    if w_like is not None and sum(a * b for a, b in zip(w, w_like)) < 0:
        w = [-x for x in w]
    A = _coefs_mp(sum(x * x for x in w))[0]
    wt = _cross(w, t)
    wwt = _cross(w, wt)
    return [t[i] - wt[i] / 2 + A * wwt[i] for i in range(3)], w


def _skew(w):
    z = mp.mpf(0)
    return mp.matrix([[z, -w[2], w[1]], [w[2], z, -w[0]], [-w[1], w[0], z]])


def _ljacinv_blocks(v, w):
    t2 = sum(x * x for x in w)
    if t2 < IDENTITY_T2:
        return mp.eye(3), mp.zeros(3, 3)
    A, B, C, D = _coefs_mp(t2)
    W, V = _skew(w), _skew(v)
    Ji = mp.eye(3) - W / 2 + A * W * W
    VW = V * W
    WV = VW.T
    WVW = WV * W
    VWW = VW * W
    Q = V / 2 + B * (WV + VW + WVW) - C * (VWW - VWW.T - 3 * WVW) + D * (WVW * W + W * WVW)
    return Ji, -(Ji * Q * Ji)


def _np3(m):
    return np.array([[float(m[i, j]) for j in range(3)] for i in range(3)])


# ---- vectorised fp64 front ends --------------------------------------------------------------------------------------------
def so3_log(q):
    q = np.asarray(q, np.float64)
    with mp.workdps(DPS):
        return np.array([[float(x) for x in _so3_log(_mpf(r))] for r in q.reshape(-1, 4)]).reshape(q.shape[:-1] + (3,))


def se3_log(q, t):
    """[..., 6] = (v, w) = log of the pose (q, t); q need not be unit (its rotation is taken)."""
    q, t = np.asarray(q, np.float64), np.asarray(t, np.float64)
    out = []
    with mp.workdps(DPS):
        for qq, tt in zip(q.reshape(-1, 4), np.broadcast_to(t, q.shape[:-1] + (3,)).reshape(-1, 3)):
            v, w = _se3_log(_mpf(qq), _mpf(tt))
            out.append([float(x) for x in v + w])
    return np.array(out).reshape(q.shape[:-1] + (6,))


def ljacinv_blocks(xi):
    """(Ji, Mi) of the SE(3) inverse left Jacobian [[Ji, Mi], [0, Ji]] at xi = (v, w); each [..., 3, 3]."""
    xi = np.asarray(xi, np.float64)
    Ji, Mi = [], []
    with mp.workdps(DPS):
        for r in xi.reshape(-1, 6):
            m = _mpf(r)
            a, b = _ljacinv_blocks(m[:3], m[3:])
            Ji.append(_np3(a)); Mi.append(_np3(b))
    shp = xi.shape[:-1] + (3, 3)
    return np.array(Ji).reshape(shp), np.array(Mi).reshape(shp)


def ljacinv(xi):
    """The 6x6 [[Ji, Mi], [0, Ji]] at xi, [..., 6, 6]."""
    Ji, Mi = ljacinv_blocks(xi)
    L = np.zeros(Ji.shape[:-2] + (6, 6))
    L[..., :3, :3] = Ji; L[..., 3:, 3:] = Ji; L[..., :3, 3:] = Mi
    return L


def quat_sub(qa, qb):
    """mju_subQuat: body-frame rotation vector taking qb to qa, angle wrapped to (-pi, pi]."""
    qa, qb = np.asarray(qa, np.float64), np.asarray(qb, np.float64)
    out = []
    with mp.workdps(DPS):
        for a, b in zip(qa.reshape(-1, 4), qb.reshape(-1, 4)):
            d = _qmul(_qconj(_mpf(b)), _mpf(a))
            s = mp.sqrt(d[1] ** 2 + d[2] ** 2 + d[3] ** 2)
            if s == 0:
                out.append([0.0] * 3)
                continue
            ang = 2 * mp.atan2(s, d[0])
            if ang > mp.pi:
                ang -= 2 * mp.pi
            out.append([float(ang / s * x) for x in d[1:]])
    return np.array(out).reshape(qa.shape[:-1] + (3,))


def quat_integrate(q, w):
    """normalize(q) * exp(w) (mju_quatIntegrate with dt folded into w), normalised."""
    q, w = np.asarray(q, np.float64), np.asarray(w, np.float64)
    out = []
    with mp.workdps(DPS):
        for qq, ww in zip(q.reshape(-1, 4), np.broadcast_to(w, q.shape[:-1] + (3,)).reshape(-1, 3)):
            a, m = _qnormalize(_mpf(qq)), _mpf(ww)
            n = mp.sqrt(sum(x * x for x in m))
            if n == 0:
                out.append([float(x) for x in a])
                continue
            k = mp.sin(n / 2) / n
            out.append([float(x) for x in _qnormalize(_qmul(a, [mp.cos(n / 2)] + [k * x for x in m]))])
    return np.array(out).reshape(q.shape)


# ---- task rows ------------------------------------------------------------------------------------------------------------
def _like(e_like, b):
    return None if e_like is None else _mpf(e_like[b, 3:])


def frame_task(pose, Jb, target, e_like=None):
    """FrameTask rows of B instances: pose [B,7] and body Jacobian Jb [B,6,nv] of the frame (the oracle's fp64 FK), target
    [B,7] (its quaternion normalised first, as the kernels do).  e = log(T_wb^-1 T_wt); J = -jlog(T_wt^-1 T_wb) Jb =
    -ljacinv(e) Jb, since log(T_wt^-1 T_wb) = -e.  e_like [B,6], a kernel's e: at theta = pi, where either sign of the
    rotation is a log (and v changes with it), take the log on the side of e_like's rotation, and evaluate J at e_like, as
    the kernels evaluate it at their own e (which also decides the side of the identity switch J lands on).
    Returns (e [B,6], J [B,6,nv])."""
    e = np.zeros((len(pose), 6))
    with mp.workdps(DPS):
        for b in range(len(pose)):
            qf, pf, tq, tp = _mpf(pose[b, :4]), _mpf(pose[b, 4:]), _qnormalize(_mpf(target[b, :4])), _mpf(target[b, 4:])
            v, w = _se3_log(_qmul(_qconj(qf), tq), _qrot(_qconj(qf), [tp[i] - pf[i] for i in range(3)]), _like(e_like, b))
            e[b] = [float(x) for x in v + w]
    return e, -ljacinv(e if e_like is None else e_like) @ Jb


def relative_frame_task(pose_f, Jb_f, pose_r, Jb_r, target, e_like=None):
    """RelativeFrameTask rows (mink/tasks/relative_frame_task.py:106-142) of frame f in root r, from both frames' poses and
    body Jacobians; target [B,7] is T_rt, the pose of the target in the root frame.  T_rf = T_wr^-1 T_wf, T_tf = T_rt^-1 T_rf,
    e = log(T_tf), J = jlog(T_tf) (Jb_f - Ad(T_rf^-1) Jb_r) with jlog(T_tf) = ljacinv(-e).  e_like as in frame_task.
    Returns (e [B,6], J [B,6,nv])."""
    B = len(pose_f)
    e = np.zeros((B, 6))
    Ad = np.zeros((B, 6, 6))
    with mp.workdps(DPS):
        for b in range(B):
            qf, pf, qr, pr = _mpf(pose_f[b, :4]), _mpf(pose_f[b, 4:]), _mpf(pose_r[b, :4]), _mpf(pose_r[b, 4:])
            tq, tp = _qnormalize(_mpf(target[b, :4])), _mpf(target[b, 4:])
            q_rf = _qmul(_qconj(qr), qf)
            t_rf = _qrot(_qconj(qr), [pf[i] - pr[i] for i in range(3)])
            v, w = _se3_log(_qmul(_qconj(tq), q_rf), _qrot(_qconj(tq), [t_rf[i] - tp[i] for i in range(3)]), _like(e_like, b))
            e[b] = [float(x) for x in v + w]
            # Ad(T_fr), T_fr = T_rf^-1: R = R_rf^T, t = -R_rf^T t_rf; Ad = [[R, [t] R], [0, R]]
            q_fr = _qconj(q_rf)
            t_fr = [-x for x in _qrot(q_fr, t_rf)]
            R = mp.matrix([_qrot(q_fr, [mp.mpf(int(i == j)) for i in range(3)]) for j in range(3)]).T
            SR = _skew(t_fr) * R
            for i in range(3):
                for j in range(3):
                    Ad[b, i, j] = Ad[b, 3 + i, 3 + j] = float(R[i, j])
                    Ad[b, i, 3 + j] = float(SR[i, j])
    return e, ljacinv(-(e if e_like is None else e_like)) @ (Jb_f - Ad @ Jb_r)
