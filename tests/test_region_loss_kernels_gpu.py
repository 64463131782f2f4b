"""GPU: the region-count entry points of csrc/losses.cu (gdrn_head_glue_fwd_ex2, gdrn_pixel_loss_fwd_ex2, gdrn_head_bwd_ex2) against
float64 autograd of the oracle's own functions (oracle/mask_oracle.py pixel losses, oracle/region_oracle.py Patch-PnP input), on
the kernels' exact inputs, in the manner of tests/test_mask_loss_kernels_gpu.py:

  * R in {2, 4, 8, 16, 32, 60, 64} x region attention on / off x mask head L1 (MO 1) / CE (MO 2) x a separate region mask or not;
  * every logit column >= N = MO + 4 + R is NaN (the output conv never writes it): all outputs stay finite and correct;
  * at R = 64 with attention the _ex2 entry points equal the _ex ones bit for bit.

Bounds as in tests/test_mask_loss_kernels_gpu.py: 1e-5 of each channel group for two-plane outputs plus one unit roundoff of the
16-bit storage format for single-plane ones; pixel losses 2e-6."""
import pytest
import torch
import torch.nn.functional as F

from loss_ref_common import HW, REPORT, check, grad_scale, nan_planes, unit_roundoff  # noqa: E402 (tests/ is on sys.path)
from oracle import mask_oracle as M

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

TOL2 = 1e-5
MODES = {"L1": 0, "CE": 2}
REGIONS = [2, 4, 8, 16, 32, 60, 64]
LOSSES = ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region")
SELECTIONS = {False: ("visib", "trunc", "visib"), True: ("visib", "trunc", "obj")}  # separate region mask or not


def tol_for(planes: int) -> float:
    return TOL2 if planes == 2 else unit_roundoff() + TOL2


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    yield
    print("worst errors:", {k: f"{v:.2e}" for k, v in sorted(REPORT.items())})


def _C():
    from gdr_net_b200.capi import C

    return C


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _n_in(R, att, with_2d):
    return 3 + 2 * with_2d + (R if att else 0)


def _ld(n_in):
    return -(-n_in // 64) * 64


def _inputs(B, R, mlt, seed):
    mo = 2 if mlt == "CE" else 1
    N = mo + 4 + R
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    z = torch.randn(B * HW, 72, device=dev, generator=g) * 2.0
    z[:, N:] = float("nan")  # never written by the output conv
    gt_xyz = torch.rand(B, 3, HW, device=dev, generator=g)
    obj = (torch.rand(B, HW, device=dev, generator=g) < 0.7).float()
    visib = obj * (torch.rand(B, HW, device=dev, generator=g) < 0.85).float()
    trunc = visib * (torch.rand(B, HW, device=dev, generator=g) < 0.9).float()
    labels = torch.randint(0, R + 1, (B, HW), device=dev, generator=g)
    labels[:, :40] = 0
    labels[:, 40:80] = R
    coord2d = torch.rand(B, 2, HW, device=dev, generator=g) * 2 - 1
    extents = torch.rand(B, 3, device=dev, generator=g) * 0.25 + 0.05
    masks = dict(obj=obj.contiguous(), visib=visib.contiguous(), trunc=trunc.contiguous())
    return dict(B=B, R=R, mlt=mlt, mo=mo, N=N, z=z.contiguous(), gt_xyz=gt_xyz, masks=masks, labels=labels.contiguous(),
                coord2d=coord2d, extents=extents)


def _ptrs(d, sel):
    return tuple(d["masks"][k].data_ptr() for k in sel)


def _ref_losses(z64, d, sel):
    B, N = d["B"], d["N"]
    head = z64[:, :N].reshape(B, 64, 64, N).permute(0, 3, 1, 2)
    m = {k: v.double().view(B, 64, 64) for k, v in d["masks"].items()}
    batch = dict(roi_xyz=d["gt_xyz"].double().view(B, 3, 64, 64), roi_mask_trunc=m["trunc"], roi_mask_visib=m["visib"],
                 roi_mask_obj=m["obj"], roi_region=d["labels"].view(B, 64, 64))
    return M.pixel_losses(head, batch, d["mlt"], sel)


def _glue_ref(z64, d, with_2d, att):
    B, mo, N = d["B"], d["mo"], d["N"]
    head = z64[:, :N].reshape(B, 64, 64, N).permute(0, 3, 1, 2)
    parts = [(head[:, mo:mo + 3] - 0.5) * d["extents"].double().view(B, 3, 1, 1)]
    if with_2d:
        parts.append(d["coord2d"].double().view(B, 2, 64, 64))
    if att:
        parts.append(F.softmax(head[:, mo + 4:], dim=1))
    return torch.cat(parts, 1).permute(0, 2, 3, 1).reshape(B * HW, -1)


def _sums(d, sel, att, ld):
    sums = torch.full((7,), float("nan"), dtype=torch.float64, device="cuda")
    _C().gdrn_pixel_loss_fwd_ex2(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), *_ptrs(d, sel), d["labels"].data_ptr(), sums.data_ptr(),
                                 d["B"], HW, MODES[d["mlt"]], d["mo"], d["R"], att, ld, _stream())
    return sums


def _finalize(sums, B):
    losses = torch.full((8,), float("nan"), device="cuda")
    vis_out = torch.full((2,), float("nan"), device="cuda")
    pose_sums = torch.zeros(4, dtype=torch.float64, device="cuda")
    vis = torch.zeros(B, 2, device="cuda")
    _C().gdrn_loss_finalize_ex(sums.data_ptr(), pose_sums.data_ptr(), vis.data_ptr(), losses.data_ptr(), vis_out.data_ptr(), B, HW, 1,
                               _stream())
    return losses


@pytest.mark.parametrize("sep", [False, True])
@pytest.mark.parametrize("mlt", list(MODES))
@pytest.mark.parametrize("R", REGIONS)
def test_pixel_loss_fwd_ex2(R, mlt, sep):
    B = 3
    d = _inputs(B, R, mlt, 100 + R + 7 * MODES[mlt])
    sel = SELECTIONS[sep]
    sums = _sums(d, sel, 1, 64 if R <= 59 else 128)
    losses = _finalize(sums, B)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(losses[:5]).all())
    L = _ref_losses(d["z"].double(), d, sel)
    for i, k in enumerate(LOSSES):
        check(f"region pixel {k}[{R},{mlt},{sep}]", losses[i:i + 1], L[k].view(1), 2e-6)


def _din(B, ld, planes, seed):
    from gdr_net_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * HW, ld, device="cuda", generator=g) * (5e-4 * grad_scale())
    return ops.PT.from_float(x, planes)


@pytest.mark.parametrize("planes", [2, 1])
@pytest.mark.parametrize("att", [1, 0])
@pytest.mark.parametrize("sep", [False, True])
@pytest.mark.parametrize("mlt", list(MODES))
@pytest.mark.parametrize("R", REGIONS)
def test_head_bwd_ex2(R, mlt, sep, att, planes):
    """d/d logits of sum_i gw_i L_i + <din, glue(logits)>, with and without din; 2-D coordinates on for planes 2, off for 1."""
    B = 3
    with_2d = int(planes == 2)
    d = _inputs(B, R, mlt, 300 + R + 7 * MODES[mlt] + 2 * att)
    mo, N = d["mo"], d["N"]
    n_in = _n_in(R, att, with_2d)
    ld = _ld(n_in)
    sel = SELECTIONS[sep]
    sums = _sums(d, sel, att, ld)
    gw = torch.tensor([0.7, -1.3, 2.1, 0.4, 1.7, 1.0, 1.0, 1.0], device="cuda") * grad_scale()
    for dmode in (None, planes):
        din = _din(B, ld, dmode, 11 + R) if dmode else None
        out = nan_planes((B * HW, 128), planes)
        _C().gdrn_head_bwd_ex2(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), *_ptrs(d, sel), d["labels"].data_ptr(), sums.data_ptr(),
                               gw.data_ptr(), din.hi_ptr if din else None, din.lo_ptr if din else None, d["extents"].data_ptr(),
                               out.hi_ptr, out.lo_ptr, B, HW, with_2d, MODES[mlt], mo, R, att, ld, _stream())
        torch.cuda.synchronize()
        z = d["z"].double().requires_grad_(True)
        L = _ref_losses(z, d, sel)
        tot = sum(float(gw[i]) * L[k] for i, k in enumerate(LOSSES))
        if din is not None:
            tot = tot + (din.float().double()[:, :n_in] * _glue_ref(z, d, with_2d, att)).sum()
        (ref,) = torch.autograd.grad(tot, z)
        got = out.float()
        assert bool(torch.isfinite(got).all())
        tag = f"[{R},{mlt},{sep},att{att},din{dmode},{planes}]"
        tol = tol_for(planes)
        check(f"region head_bwd mask{tag}", got[:, :mo], ref[:, :mo], tol)
        check(f"region head_bwd xyz{tag}", got[:, mo:mo + 3], ref[:, mo:mo + 3], tol)
        check(f"region head_bwd bg{tag}", got[:, mo + 3], ref[:, mo + 3], tol)
        check(f"region head_bwd regions{tag}", got[:, mo + 4:N], ref[:, mo + 4:N], tol)
        assert bool((out.buf[:, :, N:] == 0).all()), ("columns >= N not exactly zero", int((out.buf[:, :, N:] != 0).sum()))


@pytest.mark.parametrize("planes", [2, 1])
@pytest.mark.parametrize("with_2d", [1, 0])
@pytest.mark.parametrize("att", [1, 0])
@pytest.mark.parametrize("mlt", list(MODES))
@pytest.mark.parametrize("R", REGIONS)
def test_head_glue_fwd_ex2(R, mlt, att, with_2d, planes):
    d = _inputs(2, R, mlt, 500 + R)
    n_in = _n_in(R, att, with_2d)
    ld = _ld(n_in)
    out = nan_planes((2 * HW, ld), planes)
    _C().gdrn_head_glue_fwd_ex2(d["z"].data_ptr(), d["coord2d"].data_ptr() if with_2d else None, d["extents"].data_ptr(), out.hi_ptr,
                                out.lo_ptr, 2, HW, with_2d, d["mo"], R, att, ld, _stream())
    torch.cuda.synchronize()
    ref = _glue_ref(d["z"].double(), d, with_2d, att)
    check(f"region glue[{R},{mlt},{att},{with_2d},{planes}]", out.float()[:, :n_in], ref, tol_for(planes))
    assert bool((out.buf[:, :, n_in:] == 0).all())


@pytest.mark.parametrize("mlt", list(MODES))
def test_ex2_at_64_regions_with_attention_equals_ex(mlt):
    """The shipped head through the _ex2 entry points: sums, glue and gradient planes bit for bit those of the _ex ones."""
    B = 5
    d = _inputs(B, 64, mlt, 900 + MODES[mlt])
    C = _C()
    for sel in SELECTIONS.values():
        a = torch.full((7,), float("nan"), dtype=torch.float64, device="cuda")
        C.gdrn_pixel_loss_fwd_ex(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), *_ptrs(d, sel), d["labels"].data_ptr(), a.data_ptr(), B, HW,
                                 MODES[mlt], d["mo"], _stream())
        b = _sums(d, sel, 1, 128)
        torch.cuda.synchronize()
        assert torch.equal(a, b), (a, b)
        gw = torch.tensor([0.7, -1.3, 2.1, 0.4, 1.7, 1.0, 1.0, 1.0], device="cuda") * grad_scale()
        for with_2d in (1, 0):
            for dmode in (None, 1, 2):
                din = _din(B, 128, dmode, 5) if dmode else None
                outs = []
                for ex2 in (False, True):
                    out = nan_planes((B * HW, 128), 2)
                    args = (d["z"].data_ptr(), d["gt_xyz"].data_ptr(), *_ptrs(d, sel), d["labels"].data_ptr(), b.data_ptr(),
                            gw.data_ptr(), din.hi_ptr if din else None, din.lo_ptr if din else None, d["extents"].data_ptr(),
                            out.hi_ptr, out.lo_ptr, B, HW, with_2d, MODES[mlt], d["mo"])
                    if ex2:
                        C.gdrn_head_bwd_ex2(*args, 64, 1, 128, _stream())
                    else:
                        C.gdrn_head_bwd_ex(*args, _stream())
                    outs.append(out)
                torch.cuda.synchronize()
                assert torch.equal(outs[0].buf, outs[1].buf), (sel, with_2d, dmode)
    for with_2d in (1, 0):
        outs = []
        for ex2 in (False, True):
            out = nan_planes((B * HW, 128), 2)
            a = (d["z"].data_ptr(), d["coord2d"].data_ptr() if with_2d else None, d["extents"].data_ptr(), out.hi_ptr, out.lo_ptr, B, HW,
                 with_2d, d["mo"])
            C.gdrn_head_glue_fwd_ex2(*a, 64, 1, 128, _stream()) if ex2 else C.gdrn_head_glue_fwd_ex(*a, _stream())
            outs.append(out)
        torch.cuda.synchronize()
        assert torch.equal(outs[0].buf, outs[1].buf), with_2d
