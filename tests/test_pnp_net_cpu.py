"""Network-initialised test-time PnP (TEST.PNP_TYPE net_iter_pnp / net_ransac_pnp / net_ransac_pnp_rot), CPU part: the oracle's
restatement of OpenCV's iterative solver is pinned against the installed cv2, the oracle's mode rules against the unmodified
reference (tests/golden/pnp_net_b4.npz), and the CUDA file's logic is single-stepped on the host (one thread per CTA, tests/emu)
against the reference's own cv2 calls."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.pnp_ransac import combine_net_and_pnp  # noqa: E402
from oracle import net_pnp_oracle as N  # noqa: E402
import pnp_net_common as C  # noqa: E402  (tests/ is on sys.path: rootdir conftest)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = np.array(synth.LM_K)


def _problem(seed, n, nout, noise, off):
    """n points in front of the camera, `nout` of them with random image positions, the guess rotated by `off` rad."""
    rng = np.random.default_rng(seed)
    R, _ = cv2.Rodrigues(rng.normal(size=3))
    t = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.4, 1.5)])
    P = rng.uniform(-0.1, 0.1, (n, 3))
    uv = (P @ R.T + t) @ K.T
    uv = uv[:, :2] / uv[:, 2:] + rng.normal(scale=noise, size=(n, 2))
    uv[:nout] = rng.uniform(0, 600, (nout, 2))
    ax = rng.normal(size=3)
    rv0, _ = cv2.Rodrigues(cv2.Rodrigues(ax / np.linalg.norm(ax) * off)[0] @ R)
    return P, uv, rv0.ravel(), t + rng.normal(scale=0.02, size=3)


def test_rodrigues_restated_matches_cv2():
    rng = np.random.default_rng(0)
    vecs = [rng.normal(size=3) * s for s in (1e-9, 1e-3, 0.5, 2.0, 3.0) for _ in range(4)]
    vecs += [np.zeros(3), np.array([np.pi, 0, 0]), np.array([0, -np.pi, 0]), np.array([1, 1, 1]) / np.sqrt(3) * (np.pi - 1e-7)]
    for r in vecs:
        Rc, Jc = cv2.Rodrigues(r.reshape(3, 1))
        Ro, Jo = N.rodrigues_vec_to_mat(r)
        assert np.abs(Rc - Ro).max() < 1e-12 and np.abs(Jc - Jo).max() < 1e-9, r
        rc = cv2.Rodrigues(Rc)[0].ravel()
        ro = N.rodrigues_mat_to_vec(Rc)
        assert np.abs(rc - ro).max() < 1e-9, (r, rc, ro)
    # float32 input, as the evaluator passes the network rotation: the re-orthonormalisation matters
    for _ in range(20):
        R32 = cv2.Rodrigues(rng.normal(size=3))[0].astype(np.float32)
        assert np.abs(cv2.Rodrigues(R32.astype(np.float64))[0].ravel() - N.rodrigues_mat_to_vec(R32)).max() < 1e-9


@pytest.mark.parametrize("n", [4, 6, 300, 2000])
def test_iterative_restated_matches_cv2(n):
    """Same minimiser to 1e-9 and the same stopping point: where the last accepted step is large enough to tell, stopping one
    iteration earlier would NOT match cv2."""
    capped = 0
    for outl in (0.0, 0.2):
        for off in (0.05, 0.3, 1.0):
            for s in range(3):
                P, uv, rv0, t0 = _problem(s * 7 + n, n, int(outl * n), 0.5, off)
                rc, tc = N.pnp_iterative_cv2(P, uv, K, rv0, t0)
                ro, to, it = N.pnp_iterative_restated(P, uv, K, rv0, t0)
                assert max(np.abs(rc - ro).max(), np.abs(tc - to).max()) <= 1e-9, (outl, off, s)
                if it > 1:
                    rp, tp, _ = N.pnp_iterative_restated(P, uv, K, rv0, t0, max_iters=it - 1)
                    step = max(np.abs(rp - ro).max(), np.abs(tp - to).max())
                    if step > 1e-8:
                        assert max(np.abs(rc - rp).max(), np.abs(tc - tp).max()) > 1e-9
                capped += it == 20
    if n == 6:
        # one gross outlier among 6 points: LM creeps along a flat valley and runs into the 20-iteration cap, where cv2 stops too
        assert capped >= 2, capped


def test_oracle_matches_reference_golden(golden_dir):
    """tests/golden/pnp_net_b4.npz holds what the UNMODIFIED `GDRN_EvaluatorCustom.process_net_and_pnp` produced
    (oracle/make_golden_net_pnp.py).  The oracle's selection reproduces its point lists bit for bit, its rules + cv2 calls the
    poses (same cv2 build: exactly), and the restated LM the iterative poses within float32.  ROI 2's network translation is
    2.5 m off: the RANSAC mode falls back to it, the iterative mode keeps its own solution although it moved more than 1 m."""
    g = np.load(os.path.join(golden_dir, "pnp_net_b4.npz"))
    d = {k: torch.from_numpy(g[k]) for k in ("mask", "xyz", "coord_2d", "extents", "cams", "im_wh", "R", "t")}
    same_cv2 = str(g["cv2_version"]) == cv2.__version__
    for b in range(4):
        ip, mp = C.selected(d, b)
        assert np.array_equal(ip, g[f"img_points_{b}"]) and np.array_equal(mp, g[f"model_points_{b}"]), b
        K_b = g["cams"][b]
        for mode in C.MODES:
            want = g[f"pose_{mode}_{b}"]
            got = N.net_and_pnp(mp, ip, K_b, g["R_net"][b], g["t_net"][b], mode)
            assert np.abs(got - want).max() < (1e-9 if same_cv2 else 5e-3), (b, mode)
        got = N.net_and_pnp(mp, ip, K_b, g["R_net"][b], g["t_net"][b], "iter", solver="restated")
        assert np.abs(got - g[f"pose_iter_{b}"]).max() < 1e-5, b
    assert np.array_equal(g["pose_ransac_2"][:, 3], g["t_net"][2].astype(np.float64))
    assert np.linalg.norm(g["pose_iter_2"][:, 3] - g["t_net"][2]) > 1.0


# ------------------------------------------------------------------------------------------------ the CUDA file, single-stepped
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("g++ / CUDA headers needed for the host emulation build")
    out = tmp_path_factory.mktemp("emu") / "libpnp_net_emu.so"
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "emu", "pnp_ransac_emu.cpp"), "-o", str(out)])
    lib = ctypes.CDLL(str(out))
    lib.gdrn_pnp_ransac_workspace_bytes.restype = ctypes.c_long
    lib.gdrn_pnp_iterative_workspace_bytes.restype = ctypes.c_long
    return lib


def _run_emu(lib, d, R_net, t_net):
    """All three modes through the emulated kernels + `combine_net_and_pnp`.  Returns (poses by mode, n_points, inliers)."""
    B = d["mask"].shape[0]
    h = w = d["mask"].shape[-1]
    f = lambda t: np.ascontiguousarray(np.asarray(t, np.float32))  # noqa: E731
    mask, xyz, c2d, ext, imwh, cams = (f(d[k]) for k in ("mask", "xyz", "coord_2d", "extents", "im_wh", "cams"))
    Rn, tn = f(R_net), f(t_net)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    ws = np.zeros(lib.gdrn_pnp_iterative_workspace_bytes(B, h * w) // 8 + 1, np.float64)
    pose_it = np.zeros((B, 3, 4), np.float32)
    info_it = np.zeros((B, 4), np.int32)
    rc = lib.gdrn_pnp_iterative(P(mask), P(xyz), P(c2d), P(ext), P(imwh), P(cams), P(Rn), P(tn), B, h, w, 1, ctypes.c_float(0.5), 20,
                                P(ws), ctypes.c_long(ws.nbytes), P(pose_it), P(info_it), None)
    assert rc == 0
    ws = np.zeros(lib.gdrn_pnp_ransac_workspace_bytes(B, h * w, 20) // 8 + 1, np.float64)
    pose_rs = np.zeros((B, 3, 4), np.float32)
    info_rs = np.zeros((B, 4), np.int32)
    inl = np.zeros((B, h * w), np.uint8)
    rc = lib.gdrn_pnp_ransac(P(mask), P(xyz), P(c2d), P(ext), P(imwh), P(cams), B, h, w, 1, ctypes.c_float(0.5), ctypes.c_double(3.0), 20,
                             ctypes.c_double(0.99), P(ws), ctypes.c_long(ws.nbytes), P(pose_rs), P(info_rs), P(inl), None)
    assert rc == 0
    assert np.array_equal(info_it[:, 0], info_rs[:, 0])
    T = torch.from_numpy
    poses = {"iter": combine_net_and_pnp("iter", T(Rn), T(tn), T(pose_it), T(info_it[:, 2] != 0)).numpy()}
    for mode in ("ransac", "ransac_rot"):
        poses[mode] = combine_net_and_pnp(mode, T(Rn), T(tn), T(pose_rs), T(info_rs[:, 3] != 0)).numpy()
    return poses, info_it, inl


def test_kernel_logic_emulated_matches_cv2(emu):
    d = synth.make_pnp_maps(8, seed=0)
    R_net, t_net = C.net_pose(d, far=(3,))
    ref = C.reference_results(d, R_net, t_net)
    poses, info, inl = _run_emu(emu, d, R_net, t_net)
    assert (info[:, 1] > 0).all() and (info[:, 1] <= 20).all()
    C.check(ref, R_net, t_net, info[:, 0], poses, inl, d)


def test_kernel_logic_emulated_edge_cases(emu):
    d, R_net, t_net = C.edge_case_batch()
    ref = C.reference_results(d, R_net, t_net)
    poses, info, inl = _run_emu(emu, d, R_net, t_net)
    assert info[:4, 0].tolist() == [0, 3, 4, 8]
    assert info[:2, 2].tolist() == [0, 0] and info[2:, 2].all()  # LM runs from 4 points on
    net = np.concatenate([R_net, t_net[:, :, None]], axis=2)
    for mode in C.MODES:
        assert np.array_equal(poses[mode][:2], net[:2]), mode  # fewer than 4 points: the network pose, exactly
    assert np.array_equal(poses["ransac"][2], net[2])  # 4 points in a RANSAC mode: network pose (cv2: P3P)
    # RANSAC failed, here and in cv2 (whose rvec / tvec are then indeterminate for a float32 guess): the network pose
    assert np.array_equal(poses["ransac"][3], net[3]) and len(ref[3]["inliers"]) == 0
    assert np.array_equal(poses["ransac"][4][:, 3], t_net[4])  # te > 1 m: network translation
    assert np.linalg.norm(poses["iter"][4][:, 3] - t_net[4]) > 1.0  # ... which the iterative mode does not apply
    C.check(ref, R_net, t_net, info[:, 0], poses, inl, d, min_identical_frac=0.0)


def test_kernel_logic_emulated_matches_reference_golden(emu, golden_dir):
    g = np.load(os.path.join(golden_dir, "pnp_net_b4.npz"))
    d = {k: g[k] for k in ("mask", "xyz", "coord_2d", "extents", "cams", "im_wh")}
    poses, info, inl = _run_emu(emu, d, g["R_net"], g["t_net"])
    for b in range(4):
        assert int(info[b, 0]) == len(g[f"img_points_{b}"])
        want = g[f"pose_iter_{b}"]
        assert np.abs(poses["iter"][b] - want).max() < 1e-5, b
        for mode in ("ransac", "ransac_rot"):
            want = g[f"pose_{mode}_{b}"]
            ang = np.degrees(np.arccos(np.clip((np.trace(poses[mode][b][:, :3].astype(np.float64) @ want[:, :3].T) - 1) / 2, -1, 1)))
            assert ang < 1.0 and np.abs(poses[mode][b][:, 3] - want[:, 3]).max() < 5e-3 * want[2, 3], (b, mode, ang)
