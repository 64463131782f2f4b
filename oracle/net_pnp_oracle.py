"""CPU oracle for the network-initialised test-time PnP modes of the evaluator -- TEST INFRASTRUCTURE ONLY.

Only tests/ may import this module; the product path (gdr_net_b200/pnp_ransac.py -> csrc/pnp_ransac.cu) never does.  The
selection and the RANSAC restatement it builds on live in oracle/pnp_oracle.py.

What the reference does (`process_net_and_pnp`, core/gdrn_modeling/gdrn_evaluator.py:187-314 and
gdrn_custom_evaluator.py:207-335), per ROI on the host, for TEST.PNP_TYPE net_iter_pnp / net_ransac_pnp / net_ransac_pnp_rot:
  * points selected like `get_img_model_points_with_coords2d` (MASK_THR_TEST);
  * fewer than 4 points: the network pose;
  * rvec0 = cv2.Rodrigues(R_net) on the float32 network rotation (float32 out), tvec0 = t_net (a float32 row view);
  * "iter": cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True, rvec0, tvec0).  cv2 writes the solution INTO the float32
    guess arrays and returns them, so rvec / tvec come back rounded to float32 and `t_est` IS `trans_est_net` afterwards: the
    reference's `te(t_est, trans_est_net) > 1` fallback compares an array with itself and never fires in this mode;
  * "ransac" / "ransac_rot": cv2.solvePnPRansac(EPNP, useExtrinsicGuess=True, 3 px, 20 iterations).  EPnP ignores the guess
    (the results are bit-identical to the call without one); the outputs are new float64 arrays.  A failed call (no 5
    inliers) returns False, which the reference ignores, with rvec / tvec that are NOT the guess but the contents of an
    uninitialised buffer when the guess is float32 (observed with cv2 4.13: zeros in one call, stale values of earlier arrays in
    another), so the reference's pose is indeterminate there; the oracle and the device use the network pose.
    "ransac": t_net where te(t_pnp, t_net) > 1 m; "ransac_rot": always t_net;
  * R = cv2.Rodrigues(rvec).

`pnp_iterative_restated` restates what OpenCV runs for the iterative call (calib3d `cvFindExtrinsicCameraParams2` with
useExtrinsicGuess, driven by `CvLevMarq`), pinned against cv2 by tests/test_pnp_net_cpu.py; the CUDA kernel `pnp_lm_kernel`
follows it line by line:
  * parameters p = (rvec, tvec), residual = projection (pixels, zero distortion) - image point, 2n entries;
  * CALC_J: J and r at p; JtJ, Jtr; prev = p; p = prev - solve(JtJ with diag * (1 + 10^l), Jtr) by SVD (DECOMP_SVD, back
    substitution threshold 2 DBL_EPSILON sum(w)); on the first iteration prevErr = |r|;
  * CHECK_ERR: err = |r(p)|; if err > prevErr and ++l <= 16: re-solve from prev with the larger damping, check again;
    otherwise l = max(l - 1, -16); ++iters; stop when iters >= 20 or |p - prev| / (|prev| + DBL_EPSILON) < FLT_EPSILON;
    else prevErr = err and back to CALC_J;
  * l starts at -3; the Jacobian of R(r) is cv::Rodrigues' 3x9 derivative.
"""
from __future__ import annotations

import numpy as np

from oracle import pnp_oracle as O

DBL_EPS = float(np.finfo(np.float64).eps)
FLT_EPS = float(np.finfo(np.float32).eps)


# ------------------------------------------------------------------------------------------------ Rodrigues (cv::Rodrigues)


def rodrigues_vec_to_mat(r):
    """Vector -> (R [3,3], dRdr [3,9]): dRdr[j, k] = d R.flat[k] / d r_j, the closed forms of cv::Rodrigues."""
    r = np.asarray(r, np.float64).reshape(3)
    theta = float(np.sqrt(r @ r))
    if theta < DBL_EPS:
        J = np.zeros((3, 9))
        J[0, 5], J[0, 7], J[1, 2], J[1, 6], J[2, 1], J[2, 3] = -1, 1, 1, -1, -1, 1
        return np.eye(3), J
    c, s = np.cos(theta), np.sin(theta)
    c1 = 1.0 - c
    itheta = 1.0 / theta
    rx, ry, rz = r * itheta
    rrt = np.array([rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz])
    r_x = np.array([0, -rz, ry, rz, 0, -rx, -ry, rx, 0])
    eye = np.array([1.0, 0, 0, 0, 1, 0, 0, 0, 1])
    R = c * eye + c1 * rrt + s * r_x
    drrt = np.array([[rx + rx, ry, rz, ry, 0, 0, rz, 0, 0],
                     [0, rx, 0, rx, ry + ry, rz, 0, rz, 0],
                     [0, 0, rx, 0, 0, ry, rx, ry, rz + rz]])
    d_r_x = np.array([[0, 0, 0, 0, 0, -1, 0, 1, 0],
                      [0, 0, 1, 0, 0, 0, -1, 0, 0],
                      [0, -1, 0, 1, 0, 0, 0, 0, 0]], np.float64)
    J = np.zeros((3, 9))
    for i, ri in enumerate((rx, ry, rz)):
        a0, a1, a2 = -s * ri, (s - 2 * c1 * itheta) * ri, c1 * itheta
        a3, a4 = (c - s * itheta) * ri, s * itheta
        J[i] = a0 * eye + a1 * rrt + a2 * drrt[i] + a3 * r_x + a4 * d_r_x[i]
    return R.reshape(3, 3), J


def rodrigues_mat_to_vec(R):
    """Matrix -> vector like cv::Rodrigues: re-orthonormalise through the SVD (R = U Vt), then the axis / angle closed forms
    with OpenCV's theta ~ 0 and theta ~ pi branches."""
    _, Ut, Vt = O.jacobi_svd_cv(np.asarray(R, np.float64))
    R = Ut.T @ Vt
    rx, ry, rz = R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]
    s = np.sqrt((rx * rx + ry * ry + rz * rz) * 0.25)
    c = min(max((R[0, 0] + R[1, 1] + R[2, 2] - 1) * 0.5, -1.0), 1.0)
    theta = np.arccos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        rx = np.sqrt(max((R[0, 0] + 1) * 0.5, 0.0))
        ry = np.sqrt(max((R[1, 1] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0)
        rz = np.sqrt(max((R[2, 2] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)
        if abs(rx) < abs(ry) and abs(rx) < abs(rz) and (R[1, 2] > 0) != (ry * rz > 0):
            rz = -rz
        theta /= np.sqrt(rx * rx + ry * ry + rz * rz)
        return np.array([rx, ry, rz]) * theta
    vth = 1.0 / (2 * s) * theta
    return np.array([rx, ry, rz]) * vth


# ------------------------------------------------------------------------------------------------ iterative PnP (restated)


def _residual(p, M, m, K, want_J):
    R, dRdr = rodrigues_vec_to_mat(p[:3])
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    Xc = M @ R.T + p[3:]
    z = np.where(Xc[:, 2] != 0, 1.0 / np.where(Xc[:, 2] != 0, Xc[:, 2], 1.0), 1.0)
    x, y = Xc[:, 0] * z, Xc[:, 1] * z
    r = np.empty(2 * len(M))
    r[0::2] = fx * x + cx - m[:, 0]
    r[1::2] = fy * y + cy - m[:, 1]
    if not want_J:
        return r, None
    J = np.zeros((2 * len(M), 6))
    for j in range(3):
        dX = M @ dRdr[j, 0:3]
        dY = M @ dRdr[j, 3:6]
        dZ = M @ dRdr[j, 6:9]
        J[0::2, j] = fx * z * (dX - x * dZ)
        J[1::2, j] = fy * z * (dY - y * dZ)
    J[0::2, 3], J[0::2, 5] = fx * z, -fx * x * z
    J[1::2, 4], J[1::2, 5] = fy * z, -fy * y * z
    return r, J


def svd_solve(A, b):
    """cv::solve(A, b, DECOMP_SVD): Jacobi SVD, back substitution over the singular values above 2 DBL_EPSILON sum(w)."""
    w, Ut, Vt = O.jacobi_svd_cv(A)
    thr = w.sum() * DBL_EPS * 2
    x = np.zeros(A.shape[1])
    for j in range(len(w)):
        if abs(w[j]) > thr:
            x += (Ut[j] @ b) / w[j] * Vt[j]
    return x


def pnp_iterative_restated(model_points, image_points, K, rvec0, tvec0, max_iters=20):
    """cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) for n >= 4 points, zero distortion.
    Returns (rvec [3], tvec [3], accepted iterations)."""
    M = np.asarray(model_points, np.float64).reshape(-1, 3)
    m = np.asarray(image_points, np.float64).reshape(-1, 2)
    K = np.asarray(K, np.float64)
    p = np.concatenate([np.asarray(rvec0, np.float64).reshape(3), np.asarray(tvec0, np.float64).reshape(3)])
    lam, iters = -3, 0
    r, J = _residual(p, M, m, K, True)
    prev_err = float(np.sqrt(r @ r))
    while True:
        JtJ, Jtr, prev = J.T @ J, J.T @ r, p.copy()

        def step():
            A = JtJ.copy()
            A[np.diag_indices(6)] *= 1.0 + np.exp(lam * np.log(10.0))
            return prev - svd_solve(A, Jtr)

        p = step()
        while True:
            r, _ = _residual(p, M, m, K, False)
            err = float(np.sqrt(r @ r))
            if err > prev_err:
                lam += 1
                if lam <= 16:
                    p = step()
                    continue
            break
        lam = max(lam - 1, -16)
        iters += 1
        if iters >= max_iters or np.sqrt(((p - prev) ** 2).sum()) / (np.sqrt((prev ** 2).sum()) + DBL_EPS) < FLT_EPS:
            return p[:3], p[3:], iters
        prev_err = err
        r, J = _residual(p, M, m, K, True)


def pnp_iterative_cv2(model_points, image_points, K, rvec0, tvec0):
    """The reference's own call (gdrn_custom_evaluator.py:300-310).  rvec0 / tvec0 are passed as given (float32 in the reference:
    the solution is then written back into them in float32).  Returns (rvec, tvec) as cv2 hands them back."""
    import cv2

    rvec0 = np.array(rvec0, copy=True).reshape(3, 1)
    tvec0 = np.array(tvec0, copy=True).reshape(3)
    _, rvec, tvec = cv2.solvePnP(np.ascontiguousarray(np.asarray(model_points, np.float64)),
                                 np.ascontiguousarray(np.asarray(image_points, np.float64)), np.asarray(K, np.float64),
                                 np.zeros((8, 1)), flags=cv2.SOLVEPNP_ITERATIVE, useExtrinsicGuess=True, rvec=rvec0, tvec=tvec0)
    return rvec.reshape(3), tvec.reshape(3)


# ------------------------------------------------------------------------------------------------ the evaluator's mode rules


def net_and_pnp(model_points, image_points, K, R_net, t_net, pnp_type="iter", solver="cv2"):
    """One ROI of `process_net_and_pnp`.  R_net [3,3] / t_net [3] float32 network pose; solver "cv2" (the reference's calls) or
    "restated" (pnp_iterative_restated for "iter"; the RANSAC modes always use cv2, whose restatement is pinned elsewhere).
    A failed RANSAC gives the network pose (the reference's result is indeterminate there, see above).
    Returns the [3,4] float64 pose."""
    import cv2

    R_net = np.asarray(R_net, np.float32)
    t_net = np.asarray(t_net, np.float32).reshape(3)
    net_pose = np.concatenate([R_net, t_net.reshape(3, 1)], axis=1).astype(np.float64)
    if len(image_points) < 4:
        return net_pose
    rvec0, _ = cv2.Rodrigues(R_net)  # float32 in, float32 out
    if pnp_type == "iter":
        if solver == "cv2":
            rvec, tvec = pnp_iterative_cv2(model_points, image_points, K, rvec0, t_net)
        else:
            rvec, tvec, _ = pnp_iterative_restated(model_points, image_points, K, rvec0, t_net)
            rvec, tvec = rvec.astype(np.float32), tvec.astype(np.float32)  # written back into the float32 guess arrays
        R, _ = cv2.Rodrigues(rvec.reshape(3, 1))
        return np.concatenate([R.astype(np.float64), tvec.reshape(3, 1).astype(np.float64)], axis=1)
    if pnp_type not in ("ransac", "ransac_rot"):
        raise ValueError(pnp_type)
    p3 = np.ascontiguousarray(np.asarray(model_points, np.float64)[None])
    p2 = np.ascontiguousarray(np.asarray(image_points, np.float64)[None])
    ok, rvec, tvec, _ = cv2.solvePnPRansac(p3, p2, np.asarray(K, np.float64), np.zeros((8, 1)), flags=cv2.SOLVEPNP_EPNP,
                                          useExtrinsicGuess=True, rvec=rvec0.copy(), tvec=t_net.copy(), reprojectionError=3.0,
                                          iterationsCount=20)
    if not ok:
        return net_pose
    R, _ = cv2.Rodrigues(rvec)
    t = np.asarray(tvec, np.float64).reshape(3)
    if pnp_type == "ransac_rot" or np.linalg.norm(t_net.astype(np.float64) - t) > 1:
        t = t_net.astype(np.float64)
    return np.concatenate([np.asarray(R, np.float64), t.reshape(3, 1)], axis=1)
