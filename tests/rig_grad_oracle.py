"""Host references for the rig backward, shared by tests/test_rig_grad_host.py and tests/test_gpu_rig_grad.py:
- shim(): tests/host_shim/rig_grad_shim.cpp (the product's rig Jacobians and rig IFT built for the host), compiled once per
  process into a temporary directory (the tree may be read-only);
- the lift's and the composition's Jacobians by central differences of the lift and the composition in numpy;
- frozen_fit_rig: the C-camera form of ift_oracle.frozen_fit, the stationary point of a rig fit over a frozen set;
- last_step_cells: the cells a rig's last accepted refinement step fitted, from the CPU rig oracle (tests/rig_oracle.py);
- restate_rows: dLoss/dObj of the rig backward restated in numpy from the chain's per-rig quantities."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial.transform import Rotation

from ift_oracle import DFLIP, jp6

HERE = os.path.dirname(os.path.abspath(__file__))
N, GRID = 1600, 40
FLIP = np.array([1.0, -1.0, -1.0])
_shim = None


def shim():
    global _shim
    if _shim is None:
        so = os.path.join(tempfile.mkdtemp(prefix="rig_grad_shim_"), "librig_grad_shim.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "host_shim", "rig_grad_shim.cpp")])
        _shim = C.CDLL(so)
    return _shim


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def rot(v):
    return Rotation.from_rotvec(v).as_matrix()


def log(R):
    return Rotation.from_matrix(R).as_rotvec()


def ring(C_, seed=0):
    """cam_from_rig of a ring of C cameras (test_gpu_rig.py's): camera c turned by c * 360 / C degrees about y, with small
    random tilts, 80 mm off the rig centre."""
    rng = np.random.default_rng(seed)
    ext = np.zeros((C_, 6))
    for c in range(C_):
        R = Rotation.from_euler("xyz", [rng.normal(scale=0.03), 2 * np.pi * c / C_, rng.normal(scale=0.03)])
        ext[c, :3] = R.as_rotvec()
        ext[c, 3:] = [80.0 * np.sin(2 * np.pi * c / C_), rng.normal(scale=5.0), 80.0 * np.cos(2 * np.pi * c / C_)]
    return ext


def ext12(ext):
    """[C][12] rows (Rc row-major, tc) of cv extrinsics [C][6], as the shim reads them."""
    return np.ascontiguousarray(np.concatenate([rot(ext[:, :3]).reshape(-1, 9), ext[:, 3:]], 1))


STEPS = np.array([1e-6] * 3 + [1e-3] * 3)


def _cd(fn, x):
    """Central differences of fn: [m][6] -> [m][6] at x [m][6]: [m][6 out][6 in]."""
    out = np.zeros((len(x), 6, 6))
    for a in range(6):
        d = np.zeros(6)
        d[a] = STEPS[a]
        out[:, :, a] = (fn(x + d) - fn(x - d)) / (2 * STEPS[a])
    return out


def lift_cv(Rc, tc, v):
    """The lift of cv camera poses v [m][6] through the extrinsic (Rc, tc), as cv rig poses [m][6]."""
    R = Rc.T @ rot(v[:, :3])
    return np.concatenate([log(R), (v[:, 3:] - tc) @ Rc], 1)


def lift_jac(Rc, tc, v):
    """L = d lift / d v in the cv 6-vector, [m][6][6], by central differences."""
    return _cd(lambda x: lift_cv(Rc, tc, x), v)


def cross_jp(Rc, tc, Rc2, tc2, x):
    """jp(T_c o lift(T, E_c2)) of camera poses T given by their jp 6-vectors x [m][6]."""
    R = DFLIP @ rot(x[:, :3])
    t = x[:, 3:] * FLIP
    Rr, tr = Rc2.T @ R, (t - tc2) @ Rc2
    Rk, tk = Rc @ Rr, tr @ Rc.T + tc
    return np.concatenate([log(DFLIP @ Rk), tk * FLIP], 1)


def cross_jac(Rc, tc, Rc2, tc2, v):
    """K = d jp(T_c o lift(T, E_c2)) / d jp(T) at the cv camera poses v [m][6], [m][6][6], by central differences."""
    x = np.concatenate([log(DFLIP @ rot(v[:, :3])), v[:, 3:] * FLIP], 1)
    return _cd(lambda y: cross_jp(Rc, tc, Rc2, tc2, y), x)


def _rig_residuals(Y, uv, cam, ext, fcc, R, t):
    q = Y @ R.T
    X = q + t
    Rc, tc = rot(ext[cam, :3]), ext[cam, 3:]
    Xc = np.einsum("nij,nj->ni", Rc, X) + tc
    f, cx, cy = fcc[cam, 0], fcc[cam, 1], fcc[cam, 2]
    r = np.stack([f * Xc[:, 0] / Xc[:, 2] + cx, f * Xc[:, 1] / Xc[:, 2] + cy], 1) - uv
    return q, Xc, Rc, r


def frozen_fit_rig(Y, uv, cam, ext, fcc, R, t, iters=200):
    """Stationary point of the rig fit sum |pi_c(Rc (R Y + t) + tc) - p|^2 over the frozen set (cell i in camera cam[i]),
    by Gauss-Newton in the left chart of the rig pose, to a step below 1e-14: the C-camera form of ift_oracle.frozen_fit."""
    for _ in range(iters):
        q, Xc, Rc, r = _rig_residuals(Y, uv, cam, ext, fcc, R, t)
        dX = np.zeros((len(Y), 3, 6))
        dX[:, 0, 1], dX[:, 0, 2] = q[:, 2], -q[:, 1]
        dX[:, 1, 0], dX[:, 1, 2] = -q[:, 2], q[:, 0]
        dX[:, 2, 0], dX[:, 2, 1] = q[:, 1], -q[:, 0]
        dX[:, :, 3:] = np.eye(3)
        f, z = fcc[cam, 0], Xc[:, 2]
        g = np.zeros((len(Y), 2, 3))
        g[:, 0, 0] = f / z; g[:, 0, 2] = -f * Xc[:, 0] / z ** 2
        g[:, 1, 1] = f / z; g[:, 1, 2] = -f * Xc[:, 1] / z ** 2
        J = (g @ Rc @ dX).reshape(-1, 6)
        step = -np.linalg.solve(J.T @ J, J.T @ r.reshape(-1))
        R = rot(step[:3]) @ R
        t = t + step[3:]
        if np.abs(step).max() < 1e-14:
            break
    return R, t


def rig_ift(cam, Y, uv, ext, fcc, pose):
    """The shim's d jp6 / dY [m][6][3] of the rig fit over cells (cam, Y, uv) at the cv rig pose; None if it is not defined."""
    D = np.zeros((len(Y), 6, 3))
    ok = shim().shim_rig_ift_deriv(len(Y), p(np.ascontiguousarray(cam, np.int32)), p(np.ascontiguousarray(Y, np.float64)),
                                   p(np.ascontiguousarray(uv, np.float64)), p(ext12(ext)), p(np.ascontiguousarray(fcc, np.float64)),
                                   p(np.ascontiguousarray(pose, np.float64)), p(D))
    return D if ok else None


def last_step_cells(cfg, coords, pix, intr, ext, hyp_pose, start, steps):
    """The (camera, cell) pairs of the last accepted step of the rig's refinement from `start`, `steps` steps accepted: the
    CPU rig oracle's inlier map after `steps` steps minus that after steps - 1 (each step adds 1 to the cells it selects).
    Also the smaller of the two runs' threshold margins, and the final inlier map."""
    import rig_oracle as RO
    runs = []
    for k in (steps - 1, steps):
        cfg.ref_steps = k
        runs.append(RO.forward(cfg, coords, pix, intr, ext, hyp_pose, start=start))
    diff = runs[1]["inlier_map"] - runs[0]["inlier_map"]
    assert diff.min() >= 0 and diff.max() <= 1
    cam, cell = np.nonzero(diff)
    return cam, cell, min(r["min_margin"] for r in runs), runs[1]


def _q4(cell, fix_q4):
    x, y = cell % GRID, cell // GRID
    return cell if fix_q4 else x * GRID + y


def restate_rows(cfg, C_, coords, pix, ext, rig_hyp, sf, hyp_pose, img_idx, dpnp, dl, dref_dhyp, dref_dobj, sog):
    """dLoss/dObj [n][N * 3] of the rig backward in numpy, from the rig's dl [R][6], dRefineHyp [R][6][6], direct IFT matrix
    dref_dobj [R][6][C N 3] and score output gradients sog [R][P], the frames' dPNP [n][H][6][12], and the pass's pool
    (rig_hyp [R][P][6], sf [R][P]), hypotheses and minimal sets:
      path I direct   dl . dref_dobj into every camera frame's cells;
      path I support  sf_j dLdAvg L_j dPNP[f'][h] onto hypothesis (f', h)'s minimal set, cells row-major;
      path II direct  for every camera frame f and slot j, the soft-inlier score's derivative at T_c o T_j (the diffmap
                      error in k_score's fp32 roundings) weighted by the clamped sog_j, columns in quirk Q4's layout;
      path II support the 1x6 w[f][j] with respect to jp(T_c o T_j), summed over the rig's cameras through K_c,j and
                      applied through dPNP[f'][h] to hypothesis (f', h)'s minimal set, columns in quirk Q4's layout.
    L and K are central differences of the lift and the composition, the score derivative is written from the projection
    in the jp frame (not from the product's formulas), and the rotation's derivative is a central difference of exp."""
    f, cx, cy = cfg.focal, cfg.cx, cfg.cy
    thr, alpha, beta, clamp, fix_q4 = float(cfg.thr2d), cfg.alpha, cfg.beta, cfg.grad_clamp, cfg.fix_q4
    n, H = hyp_pose.shape[:2]
    R_, P = n // C_, C_ * H
    rows = np.zeros((n, N * 3))
    dldavg = np.einsum("rk,rki->ri", dl, dref_dhyp.reshape(R_, 6, 6))
    Rcs = rot(ext[:, :3])
    # path I direct
    for r in range(R_):
        rows[r * C_:(r + 1) * C_] += (dl[r] @ dref_dobj[r].reshape(6, C_ * N * 3)).reshape(C_, N * 3)
    # path II: w and the direct part, per camera frame
    W = np.zeros((n, P, 6))
    for fr in range(n):
        r, c = divmod(fr, C_)
        Rr, tr = rot(rig_hyp[r, :, :3]), rig_hyp[r, :, 3:]
        Rk, tk = Rcs[fr] @ Rr, tr @ Rcs[fr].T + ext[fr, 3:]
        Rj, tj = DFLIP @ Rk, tk * FLIP                                # [P][3][3], [P][3] in jp
        go = sog[r] if clamp <= 0 else np.clip(sog[r], -clamp, clamp)
        Yw = coords[fr].astype(np.float32).astype(np.float64)          # [N][3]
        pu = pix[fr, :, 0].astype(np.float32).astype(np.float64)
        pv = pix[fr, :, 1].astype(np.float32).astype(np.float64)
        X, Y, Z = Yw[:, 0], Yw[:, 1], Yw[:, 2]
        # the reprojection error of the diffmap, with k_score's roundings, in the cv pose of the same camera pose
        xc = ((Rj[:, 0, 0, None] * X + Rj[:, 0, 1, None] * Y) + Rj[:, 0, 2, None] * Z) + tj[:, 0, None]
        yc = ((-Rj[:, 1, 0, None] * X + -Rj[:, 1, 1, None] * Y) + -Rj[:, 1, 2, None] * Z) + -tj[:, 1, None]
        zc = ((-Rj[:, 2, 0, None] * X + -Rj[:, 2, 1, None] * Y) + -Rj[:, 2, 2, None] * Z) + -tj[:, 2, None]
        iz = np.where(zc != 0, 1.0 / np.where(zc != 0, zc, 1.0), 1.0)
        pfu, pfv = ((xc * iz) * f + cx).astype(np.float32), ((yc * iz) * f + cy).astype(np.float32)
        du, dv = (pu.astype(np.float32) - pfu).astype(np.float64), (pv.astype(np.float32) - pfv).astype(np.float64)
        e = np.minimum(np.sqrt(du * du + dv * dv), 100.0).astype(np.float32).astype(np.float64)
        sg = 1.0 / (1.0 + np.exp(-beta * (thr - e)))
        g = go[:, None] * (-alpha * beta * sg * (1.0 - sg))            # [P][N] d score / d error
        # the error's derivative through the jp projection
        Xj = np.einsum("pik,nk->pni", Rj, Yw) + tj[:, None, :]
        ex, ey, ez = Xj[..., 0], Xj[..., 1], Xj[..., 2]
        ok = np.abs(ez) >= 1e-8
        ez = np.where(ok, ez, 1.0)
        px, py = -f * ex / ez + cx, f * ey / ez + cy
        ddx, ddy = pu - px, pv - py
        err = np.sqrt(ddx * ddx + ddy * ddy)
        ok &= err <= 100.0
        a0, a1 = -ddx / (err + 1e-8), -ddy / (err + 1e-8)              # d error / d (px, py), as k_dscore regularises it
        G = np.stack([a0 * (-f / ez), a1 * (f / ez), a0 * (f * ex / ez ** 2) + a1 * (-f * ey / ez ** 2)], -1)
        G *= np.where(ok, g, 0.0)[..., None]                            # [P][N][3] d score / d X_jp
        acc = np.einsum("pni,pik->nk", G, Rj)                           # d / dY
        cols = _q4(np.arange(N), fix_q4)
        rows[fr].reshape(N, 3)[cols] += acc
        rod = log(Rj)
        W[fr, :, 3:] = G.sum(1)
        for m in range(3):
            d = np.zeros(3)
            d[m] = 1e-7
            dR = (rot(rod + d) - rot(rod - d)) / 2e-7                   # [P][3][3]
            W[fr, :, m] = np.einsum("pni,pik,nk->p", G, dR, Yw)
    # the support scatters
    for fr in range(n):
        r, c2 = divmod(fr, C_)
        L = lift_jac(Rcs[fr], ext[fr, 3:], hyp_pose[fr])               # [H][6][6]
        u2 = np.zeros((H, 6))
        for c in range(C_):
            K = cross_jac(Rcs[r * C_ + c], ext[r * C_ + c, 3:], Rcs[fr], ext[fr, 3:], hyp_pose[fr])
            u2 += np.einsum("hk,hkm->hm", W[r * C_ + c, c2 * H:(c2 + 1) * H], K)
        u1 = sf[r, c2 * H:(c2 + 1) * H, None] * np.einsum("k,hkm->hm", dldavg[r], L)
        s1 = np.einsum("hk,hkq->hq", u1, dpnp[fr])                      # [H][12]
        s2 = np.einsum("hk,hkq->hq", u2, dpnp[fr])
        for h in range(H):
            for q in range(4):
                cell = img_idx[fr, h, q]
                if cell < 0:
                    continue
                rows[fr, cell * 3:cell * 3 + 3] += s1[h, q * 3:q * 3 + 3]
                col = _q4(cell, fix_q4) * 3
                rows[fr, col:col + 3] += s2[h, q * 3:q * 3 + 3]
    return rows, dldavg
