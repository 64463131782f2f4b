"""CPU: the mask-head switches (ROT_HEAD.MASK_LOSS_TYPE L1 | BCE | CE and the GT mask of each per-pixel loss, GDRN.py:339-400).

  * the oracle restatement (oracle/mask_oracle.py) against the unmodified reference built with those switches
    (tests/golden/train_mask_{bce,ce}_b4.npz, oracle/make_golden_masks.py);
  * `build_model_optimizer` accepts every supported combination, sizes the output conv 68 + MO rows, and rejects the rest;
  * the generalised loss entry points are declared and exported with the argument lists the engine passes;
  * the CE selection (mask_mode 3) of csrc/pnp_ransac.cu's gather kernel, single-stepped on the host (tests/emu), picks exactly
    the reference's points, ties included (tests/golden/pnp_ce_select_b3.npz)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gdr_net_b200 import synth
from oracle import gdrn_oracle as O
from oracle import mask_oracle as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name -> (ROT_HEAD switches, weight seed, batch seed), as in oracle/make_golden_masks.py
CASES = {
    "bce": (dict(MASK_LOSS_TYPE="BCE", MASK_LOSS_GT="visib", XYZ_LOSS_MASK_GT="obj"), 5, 23),
    "ce": (dict(MASK_LOSS_TYPE="CE", MASK_LOSS_GT="obj", REGION_LOSS_MASK_GT="trunc"), 6, 29),
}


def mask_config(device="cpu", **switches):
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device=device)
    for k, v in switches.items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    return cfg


def mask_gt(cfg):
    r = cfg.MODEL.CDPN.ROT_HEAD
    return (r.XYZ_LOSS_MASK_GT, r.MASK_LOSS_GT, r.REGION_LOSS_MASK_GT)


def seeded_weights(cfg, seed):
    """The reference's seeded weights: synth.seeded_state_dict seeds every tensor by its name, and the state_dict names and
    shapes of build_model_optimizer's model are the reference's."""
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(cfg)
    return synth.seeded_state_dict(model.state_dict(), seed=seed)


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    switches, wseed, bseed = CASES[case]
    g = np.load(os.path.join(golden_dir, f"train_mask_{case}_b4.npz"))
    cfg = mask_config(**switches)
    sd = seeded_weights(mask_config(**switches), wseed)
    batch = synth.make_batch(4, seed=bseed)
    mlt = switches["MASK_LOSS_TYPE"]
    # eval-mode head and pose: the same CPU ops in the same order as the reference, so bit-identical
    with torch.no_grad():
        o = M.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=False, do_loss=False, mask_loss_type=mlt)
    assert o["head"].shape[1] == 68 + M.mask_channels(mlt)
    assert np.array_equal(o["head"][:, :, ::4, ::4].numpy(), g["eval/head"])
    assert np.array_equal(o["trans"].numpy(), g["eval/trans"])
    assert np.abs(o["rot"].numpy() - g["eval/rot"]).max() <= 1e-12  # float64 numpy decode in both
    # train-mode losses: bit-identical; gradients: the oracle's autograd graph is the reference's up to the order in which
    # autograd accumulates the contributions of a tensor used twice, bounded by 5e-6 of each gradient's maximum
    leaf = O.leaf_state_dict(sd)
    o = M.gdrn_forward(leaf, batch, train=True, do_loss=True, mask_loss_type=mlt, mask_gt=mask_gt(cfg), update_stats=True)
    assert list(o["losses"]) == [k[len("loss/"):] for k in g.files if k.startswith("loss/")]
    for k, v in o["losses"].items():
        assert float(v.detach()) == float(g["loss/" + k]), (k, float(v.detach()), float(g["loss/" + k]))
    sum(o["losses"].values()).backward()
    for key in g.files:
        if key.startswith("grad/"):
            name = key[len("grad/"):]
            ref = g[key]
            err = np.abs(leaf[name].grad.numpy() - ref).max() / np.abs(ref).max()
            print(case, name, f"{err:.2e}")
            assert err <= 5e-6, (name, err)


def test_oracle_default_switches_are_gdrn_oracle():
    """With the shipped switches the restatement is gdrn_oracle.gdrn_losses itself, bit for bit."""
    batch = synth.make_batch(2, seed=3)
    g = torch.Generator().manual_seed(1)
    head = torch.randn(2, 69, 64, 64, generator=g)
    rot = O.quat2mat(torch.nn.functional.normalize(torch.randn(2, 4, generator=g), dim=1))
    t = torch.randn(2, 3, generator=g)
    a = O.gdrn_losses(head, rot, t, batch)
    b = M.gdrn_losses(head, rot, t, batch)
    assert list(a) == list(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_ce_mask_loss_truncates_soft_targets():
    """CrossEntropyLoss(out_mask, gt_mask.long()): a soft target of 0.7 is class 0, 1.0 is class 1 (GDRN.py:382-383)."""
    z = torch.tensor([[[[0.3]], [[1.2]]]])  # [1, 2, 1, 1]
    head = torch.cat([z, torch.zeros(1, 68, 1, 1)], 1)
    batch = dict(roi_xyz=torch.zeros(1, 3, 1, 1), roi_mask_trunc=torch.tensor([[[0.7]]]), roi_mask_visib=torch.ones(1, 1, 1),
                 roi_mask_obj=torch.tensor([[[1.0]]]), roi_region=torch.zeros(1, 1, 1, dtype=torch.long))
    L07 = M.pixel_losses(head, batch, "CE", ("visib", "trunc", "visib"))["loss_mask"]
    L1 = M.pixel_losses(head, batch, "CE", ("visib", "obj", "visib"))["loss_mask"]
    lse = torch.logsumexp(z.view(2), 0)
    assert torch.allclose(L07, lse - 0.3) and torch.allclose(L1, lse - 1.2)


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("mlt", ["L1", "BCE", "CE"])
def test_build_model_accepts_mask_heads(mlt):
    from gdr_net_b200 import GDRN as G

    for sel in [("visib", "trunc", "visib"), ("obj", "visib", "trunc"), ("trunc", "obj", "obj")]:
        cfg = mask_config(MASK_LOSS_TYPE=mlt, XYZ_LOSS_MASK_GT=sel[0], MASK_LOSS_GT=sel[1], REGION_LOSS_MASK_GT=sel[2])
        model, _ = G.build_model_optimizer(cfg)
        rows = 70 if mlt == "CE" else 69
        assert tuple(model.rot_head_net.features[23].weight.shape) == (rows, 256, 1, 1)
        assert tuple(model.rot_head_net.features[23].bias.shape) == (rows,)
        assert model.mask_out_dim == rows - 68


def test_ce_state_dict_has_the_reference_shapes():
    """A reference CE checkpoint loads: same keys, the output conv 70 x 256."""
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(mask_config(MASK_LOSS_TYPE="CE"))
    sd = seeded_weights(mask_config(MASK_LOSS_TYPE="CE"), 6)
    missing, unexpected = model.load_state_dict(sd, strict=True)
    assert not missing and not unexpected


@pytest.mark.parametrize("key,value", [("MASK_LOSS_GT", "gt"), ("XYZ_LOSS_MASK_GT", "full"), ("REGION_LOSS_MASK_GT", "gt"),
                                       ("MASK_LOSS_TYPE", "SmoothL1")])
def test_build_model_rejects_unknown_mask_switches(key, value):
    """The config comment lists "gt" for MASK_LOSS_GT, but gdrn_loss's gt_masks has no such key (GDRN.py:339): rejected at
    build time with the offending switch named."""
    from gdr_net_b200 import GDRN as G

    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(mask_config(**{key: value}))
    assert key in str(e.value) or "mask" in str(e.value)


# ------------------------------------------------------------------------------------------------ C ABI
def test_generalised_loss_entry_points_declared_and_exported():
    from gdr_net_b200 import capi

    protos = capi.parse_header()
    want = {"gdrn_head_glue_fwd_ex": 10, "gdrn_pixel_loss_fwd_ex": 12, "gdrn_head_bwd_ex": 19, "gdrn_loss_finalize_ex": 9,
            "gdrn_head_glue_fwd": 9, "gdrn_pixel_loss_fwd": 9, "gdrn_head_bwd": 16, "gdrn_loss_finalize": 9}
    for name, nargs in want.items():
        assert name in protos and len(protos[name][1]) == nargs, (name, protos.get(name))
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = ctypes.CDLL(capi.LIB_PATH)
    for name in want:
        assert hasattr(dll, name), name


def test_unsupported_mask_head_is_an_argument_error():
    from gdr_net_b200 import capi

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    for mode, mo in ((0, 2), (1, 2), (2, 1), (3, 1)):
        rc = dll.gdrn_pixel_loss_fwd_ex(None, None, None, None, None, None, None, 1, 4096, mode, mo, None)
        assert rc == -1 and b"mask head" in dll.gdrn_last_error(), (mode, mo)
    rc = dll.gdrn_head_glue_fwd_ex(None, None, None, None, None, 1, 4096, 0, 3, None)
    assert rc == -1 and b"mask_out" in dll.gdrn_last_error()


# ------------------------------------------------------------------------------------------------ CE selection on the host
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("g++ / CUDA headers needed for the host emulation build")
    out = tmp_path_factory.mktemp("emu") / "libpnp_ce_emu.so"
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-I/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "emu", "pnp_ransac_emu.cpp"), "-o", str(out)])
    lib = ctypes.CDLL(str(out))
    lib.gdrn_pnp_ransac_workspace_bytes.restype = ctypes.c_long
    return lib


def _gather_emu(lib, g, mode=3, thr=0.5):
    """gdrn_pnp_ransac on the host; returns the gathered points (workspace head: [B][HW][5] = X, Y, Z, u, v) and the counts."""
    B, _, h, w = g["mask"].shape
    f = lambda a: np.ascontiguousarray(np.asarray(a, np.float32))  # noqa: E731
    mask, xyz, c2d, ext, imwh, cams = f(g["mask"]), f(g["xyz"]), f(g["coord_2d"]), f(g["extents"]), f(g["im_wh"]), f(g["cams"])
    iters = 5
    nb = lib.gdrn_pnp_ransac_workspace_bytes(B, h * w, iters)
    ws = np.zeros(nb // 8 + 1, np.float64)
    pose = np.zeros((B, 3, 4), np.float32)
    info = np.zeros((B, 4), np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = lib.gdrn_pnp_ransac(P(mask), P(xyz), P(c2d), P(ext), P(imwh), P(cams), B, h, w, mode, ctypes.c_float(thr), ctypes.c_double(3.0),
                             iters, ctypes.c_double(0.99), P(ws), ctypes.c_long(ws.nbytes), P(pose), P(info), None, None)
    assert rc == 0
    return ws[:B * h * w * 5].reshape(B, h * w, 5), info[:, 0]


def test_ce_selection_oracle_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "pnp_ce_select_b3.npz"))
    for b in range(g["mask"].shape[0]):
        assert np.array_equal(M.ce_mask(g["mask"][b]), g["out_mask"][b, 0].astype(np.float32))
        W, H = int(g["im_wh"][b, 0]), int(g["im_wh"][b, 1])
        ip, mp = M.select_points_ce(g["mask"][b], g["xyz"][b], g["coord_2d"][b], g["extents"][b], W, H)
        assert np.array_equal(ip, g[f"img_points_{b}"]) and np.array_equal(mp, g[f"model_points_{b}"])


def test_ce_selection_emulated_matches_reference_golden(emu, golden_dir):
    """mask_mode 3 reads [B][2][HW] and selects z1 > z0: every tied pixel (1024 per ROI, many on the object) is class 0 and
    is dropped, exactly as get_out_mask's argmax does."""
    g = np.load(os.path.join(golden_dir, "pnp_ce_select_b3.npz"))
    pts, counts = _gather_emu(emu, g)
    for b in range(g["mask"].shape[0]):
        ip, mp = g[f"img_points_{b}"], g[f"model_points_{b}"]
        n = len(ip)
        assert int(counts[b]) == n, (b, int(counts[b]), n)
        assert np.array_equal(pts[b, :n, 0:3].astype(np.float32), mp)
        assert np.array_equal(pts[b, :n, 3:5].astype(np.float32), ip)
        # the ties matter: breaking them towards class 1 would select more points
        tie_on = g["tie"][b] & (g["xyz"][b].sum(0) > 0)  # tied pixels on the object
        assert tie_on.sum() > 100
