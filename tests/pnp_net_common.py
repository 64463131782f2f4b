"""Shared checks of the network-initialised PnP tests (TEST.PNP_TYPE net_iter_pnp / net_ransac_pnp / net_ransac_pnp_rot): the
same batch of synthetic head outputs and network poses goes through (a) the reference's per-ROI rules with its own cv2 calls
(oracle/net_pnp_oracle.py) and (b) the implementation under test (the CUDA kernels on the GPU, or their one-thread host emulation
in the CPU suite), combined by `gdr_net_b200.pnp_ransac.combine_net_and_pnp`."""
import cv2
import numpy as np
import torch

from gdr_net_b200 import synth
from oracle import net_pnp_oracle as N
from oracle import pnp_oracle as O

MODES = ("iter", "ransac", "ransac_rot")


def net_pose(d, seed=1, far=()):
    """The true pose perturbed by a seeded rotation (0.05-1 rad) and translation (2 cm); ROIs in `far` are 2.5 m too far."""
    rng = np.random.default_rng(seed)
    B = d["R"].shape[0]
    R = np.zeros((B, 3, 3), np.float32)
    t = np.zeros((B, 3), np.float32)
    for b in range(B):
        ax = rng.normal(size=3)
        ax *= rng.uniform(0.05, 1.0) / np.linalg.norm(ax)
        R[b] = (cv2.Rodrigues(ax)[0] @ d["R"][b].double().numpy()).astype(np.float32)
        t[b] = (d["t"][b].double().numpy() + rng.normal(scale=0.02, size=3)).astype(np.float32)
    for b in far:
        t[b, 2] += 2.5
    return R, t


def edge_case_batch():
    """6 ROIs: 0 no points, 1 three points, 2 four points, 3 eight points with random coordinates (RANSAC finds no 5 inliers),
    4 network translation 2.5 m off, 5 ordinary."""
    d = synth.make_pnp_maps(6, seed=5)
    d["mask"][0] = 0.0  # constant mask -> min-max normalisation is 0/0 -> nothing selected
    for b, n_keep, step in ((1, 3, 11), (2, 4, 23), (3, 8, 17)):
        ys, xs = np.nonzero((d["mask"][b, 0] > 0.5).numpy() & (d["xyz"][b].sum(0) > 0).numpy())
        m = torch.full((64, 64), 0.05)
        g = torch.Generator().manual_seed(b)
        for k in range(n_keep):
            m[ys[k * step], xs[k * step]] = 0.9
            if b == 3:
                d["xyz"][b, :, ys[k * step], xs[k * step]] = 0.05 + 0.9 * torch.rand(3, generator=g)
        d["mask"][b, 0] = m
    R_net, t_net = net_pose(d, seed=4, far=(4,))
    return d, R_net, t_net


def geodesic_deg(Ra, Rb):
    return float(np.degrees(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1.0) / 2.0, -1.0, 1.0))))


def selected(d, b):
    m = d["mask"][b, 0]
    m = (m - m.min()) / (m.max() - m.min())
    W, H = int(d["im_wh"][b, 0]), int(d["im_wh"][b, 1])
    return O.select_points(np.asarray(m, np.float32), d["xyz"][b].numpy(), d["coord_2d"][b].numpy(), d["extents"][b].numpy(), W, H)


def reference_results(d, R_net, t_net):
    """Per ROI: dict(n, mode -> reference pose [3,4], "inliers" -> cv2's RANSAC(20 iterations) inlier indices or None)."""
    out = []
    for b in range(d["mask"].shape[0]):
        ip, mp = selected(d, b)
        K = d["cams"][b].numpy()
        r = dict(n=len(ip), inliers=None)
        for mode in MODES:
            r[mode] = N.net_and_pnp(mp, ip, K, R_net[b], t_net[b], mode)
        if len(ip) >= 5:
            r["inliers"] = O.pnp_ransac_cv2(mp, ip, K, iters=20)[1]
        out.append(r)
    return out


def check(ref, R_net, t_net, n_points, poses, inliers, d, min_identical_frac=0.5, max_bad=0, verbose=True):
    """poses: mode -> [B,3,4] from the implementation under test, n_points [B], inliers [B,HW] flags of its RANSAC (20 iterations),
    d the batch (true pose R, t).

    * "iter": equal to the reference within float32 (1e-5 on R and on t in metres) everywhere;
    * RANSAC modes: within float32 where the inlier set equals cv2's (otherwise within 1 deg / 0.5 % of the depth, see
      tests/pnp_common.py), or not further from the TRUE pose than cv2's answer (+ 0.3 deg, + 0.5 % of the depth), except on at
      most `max_bad` ROIs: with 20 iterations on 30 % outliers the round-off chaotic 5-point hypotheses sometimes give the device
      and cv2 different consensus sets of different quality, in either direction (measured: 6 of 64 ROIs worse, 2 better than cv2's answer); on average the device is to be no further from the truth; n == 4: the network pose (cv2 runs P3P there; no device P3P); fewer than 4 points: the network pose."""
    B = len(ref)
    identical = valid = 0
    bad = set()
    err_mine, err_cv = [], []
    for b in range(B):
        r = ref[b]
        assert int(n_points[b]) == r["n"], (b, int(n_points[b]), r["n"])
        net = np.concatenate([R_net[b], t_net[b].reshape(3, 1)], axis=1).astype(np.float64)
        for mode in MODES:
            p = poses[mode][b].astype(np.float64)
            want = r[mode]
            if mode != "iter" and r["n"] == 4:
                want = net
            if mode == "iter" or r["inliers"] is None or r["n"] < 5:
                dR, dt = np.abs(p[:, :3] - want[:, :3]).max(), np.abs(p[:, 3] - want[:, 3]).max()
                if verbose:
                    print(f"roi {b} {mode}: points {r['n']} |dR| {dR:.1e} |dt| {dt:.1e}")
                assert dR < 1e-5 and dt < 1e-5, (b, mode, dR, dt)
                continue
            mine = np.nonzero(inliers[b])[0]
            same = np.array_equal(mine, r["inliers"])
            ang = geodesic_deg(p[:, :3], want[:, :3])
            dR, dt = np.abs(p[:, :3] - want[:, :3]).max(), np.abs(p[:, 3] - want[:, 3]).max()
            if verbose:
                print(f"roi {b} {mode}: points {r['n']} identical inliers {same} |dR| {dR:.1e} |dt| {dt:.1e} angle {ang:.4f} deg")
            if mode == "ransac":
                identical += same
                valid += 1
            if same:
                assert dR < 1e-5 and dt < 1e-5, (b, mode, dR, dt)
            R_true, t_true = d["R"][b].double().numpy(), d["t"][b].double().numpy()
            a_mine, a_cv = geodesic_deg(p[:, :3], R_true), geodesic_deg(want[:, :3], R_true)
            if mode == "ransac":
                err_mine.append(a_mine)
                err_cv.append(a_cv)
            if ang < 1.0 and dt < 5e-3 * abs(want[2, 3]):
                continue
            e_mine, e_cv = np.abs(p[:, 3] - t_true).max(), np.abs(want[:, 3] - t_true).max()
            if verbose:
                print(f"    to truth: {a_mine:.3f} deg {e_mine:.2e} m (cv2 {a_cv:.3f} deg {e_cv:.2e} m)")
            if mode == "ransac_rot":
                e_mine = e_cv
            if not (a_mine < a_cv + 0.3 and e_mine < e_cv + 5e-3 * abs(want[2, 3])):
                bad.add(b)
    assert identical >= min_identical_frac * valid, (identical, valid)
    assert len(bad) <= max_bad, sorted(bad)
    if err_cv:  # and no worse than cv2 on average
        assert np.mean(err_mine) <= 1.1 * np.mean(err_cv) + 0.1, (np.mean(err_mine), np.mean(err_cv))
        if verbose:
            print(f"mean rotation error to the truth, RANSAC mode: {np.mean(err_mine):.3f} deg (cv2 {np.mean(err_cv):.3f} deg)")
