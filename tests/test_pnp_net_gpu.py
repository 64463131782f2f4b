"""Network-initialised PnP on the device (TEST.PNP_TYPE net_iter_pnp / net_ransac_pnp / net_ransac_pnp_rot) against the reference's
own host path: cv2.solvePnP(ITERATIVE, useExtrinsicGuess) / cv2.solvePnPRansac(EPNP, 3 px, 20 iterations) on the points
selected like gdrn_evaluator.py:89-126, with the rules of `process_net_and_pnp`.  Same checks as the host emulation in the CPU
suite (tests/pnp_net_common.py)."""
import time
import types

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

import pnp_net_common as C  # noqa: E402  (tests/ is on sys.path: rootdir conftest)
from gdr_net_b200 import synth  # noqa: E402

pytestmark = pytest.mark.gpu


def _out_dict(d, R_net, t_net):
    c = lambda t: torch.as_tensor(t).cuda()  # noqa: E731
    return dict(mask=c(d["mask"]), coor_x=c(d["xyz"][:, 0:1]), coor_y=c(d["xyz"][:, 1:2]), coor_z=c(d["xyz"][:, 2:3]),
                rot=c(R_net), trans=c(t_net))


def _run(d, R_net, t_net):
    from gdr_net_b200.pnp_ransac import pnp_ransac, process_net_and_pnp

    od = _out_dict(d, R_net, t_net)
    args = (od, d["coord_2d"].cuda(), d["extents"].cuda(), d["im_wh"].cuda(), d["cams"].cuda())
    poses = {m: process_net_and_pnp(*args, pnp_type=m).cpu().numpy() for m in C.MODES}
    xyz = torch.cat([od["coor_x"], od["coor_y"], od["coor_z"]], dim=1)
    res = pnp_ransac(od["mask"], xyz, *args[1:], iters=20, return_inliers=True)
    return poses, res["num_points"].cpu().numpy(), res["inliers"].cpu().numpy()


@pytest.mark.parametrize("B,kw", [(16, {}), (64, dict(noise=0.008, outlier_frac=0.3))])
def test_net_pnp_matches_cv2(B, kw):
    d = synth.make_pnp_maps(B, seed=21, **kw)
    R_net, t_net = C.net_pose(d, seed=B, far=(3,))
    ref = C.reference_results(d, R_net, t_net)
    poses, n, inl = _run(d, R_net, t_net)
    C.check(ref, R_net, t_net, n, poses, inl, d, min_identical_frac=0.4, max_bad=B // 8, verbose=True)
    poses_b, n_b, inl_b = _run(d, R_net, t_net)
    for m in C.MODES:
        assert np.array_equal(poses[m], poses_b[m]), m  # bit-reproducible


def test_net_pnp_edge_cases():
    from gdr_net_b200.pnp_ransac import pnp_iterative

    d, R_net, t_net = C.edge_case_batch()
    ref = C.reference_results(d, R_net, t_net)
    poses, n, inl = _run(d, R_net, t_net)
    assert n[:4].tolist() == [0, 3, 4, 8]
    net = np.concatenate([R_net, t_net[:, :, None]], axis=2)
    for m in C.MODES:
        assert np.array_equal(poses[m][:2], net[:2]), m
    assert np.array_equal(poses["ransac"][2], net[2]) and np.array_equal(poses["ransac"][3], net[3])
    assert np.array_equal(poses["ransac"][4][:, 3], t_net[4]) and np.linalg.norm(poses["iter"][4][:, 3] - t_net[4]) > 1.0
    C.check(ref, R_net, t_net, n, poses, inl, d, min_identical_frac=0.0)
    c = lambda t: torch.as_tensor(t).cuda()  # noqa: E731
    res = pnp_iterative(c(d["mask"]), c(d["xyz"]), c(d["coord_2d"]), c(d["extents"]), c(d["im_wh"]), c(d["cams"]), c(R_net), c(t_net))
    assert res["ok"].cpu().tolist() == [False, False, True, True, True, True]
    it = res["iterations"].cpu().numpy()
    assert (it[:2] == 0).all() and (it[2:] >= 1).all() and (it[2:] <= 20).all()


def _cfg(pnp_type):
    rot_head = types.SimpleNamespace(MASK_LOSS_TYPE="L1", MASK_THR_TEST=0.5)
    return types.SimpleNamespace(TEST=types.SimpleNamespace(PNP_TYPE=pnp_type),
                                 MODEL=types.SimpleNamespace(CDPN=types.SimpleNamespace(ROT_HEAD=rot_head)))


def test_process_pnp_dispatch_graph_capture_and_times():
    from gdr_net_b200.pnp_ransac import process_pnp

    B = 64
    d = synth.make_pnp_maps(B, seed=2)
    R_net, t_net = C.net_pose(d, seed=7)
    od = _out_dict(d, R_net, t_net)
    args = (od, d["coord_2d"].cuda(), d["extents"].cuda(), d["im_wh"].cuda(), d["cams"].cuda())
    with pytest.raises(NotImplementedError):
        process_pnp(_cfg("net_pnp"), *args)
    ref = C.reference_results(d, R_net, t_net)  # also the host timing of the reference's cv2 loop below
    for pnp_type in ("ransac_pnp", "NET_ITER_PNP", "net_ransac_pnp", "Net_Ransac_Pnp_Rot"):
        cfg = _cfg(pnp_type)
        eager = process_pnp(cfg, *args)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            process_pnp(cfg, *args)  # warm-up on a side stream before capture
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            captured = process_pnp(cfg, *args)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(captured, eager), pnp_type
        for _ in range(3):
            process_pnp(cfg, *args)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(20):
            process_pnp(cfg, *args)
        ev1.record()
        torch.cuda.synchronize()
        dev_ms = ev0.elapsed_time(ev1) / 20
        mode = {"ransac_pnp": None, "net_iter_pnp": "iter", "net_ransac_pnp": "ransac", "net_ransac_pnp_rot": "ransac_rot"}[pnp_type.lower()]
        host = ""
        if mode is not None:
            from oracle import net_pnp_oracle as N

            t0 = time.perf_counter()
            for b in range(B):
                ip, mp = C.selected(d, b)
                N.net_and_pnp(mp, ip, d["cams"][b].numpy(), R_net[b], t_net[b], mode)
            host = f", host cv2 loop (selection + PnP, same ROIs) {1e3 * (time.perf_counter() - t0):.1f} ms"
        print(f"{pnp_type}: {dev_ms:.2f} ms per {B}-ROI batch on the device (CUDA events, 20 calls){host}")
    assert len(ref) == B
