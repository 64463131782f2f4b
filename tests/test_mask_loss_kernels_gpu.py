"""GPU: the generalised per-pixel loss kernels of csrc/losses.cu (gdrn_pixel_loss_fwd_ex, gdrn_head_bwd_ex, gdrn_head_glue_fwd_ex,
gdrn_loss_finalize_ex) against float64 autograd of the oracle's own functions (oracle/mask_oracle.py, pinned to the reference by
tests/test_mask_heads_cpu.py), in every mask head the engine launches:

  * mask loss L1 / BCE with one mask logit, CE with two (MO = 2 shifts xyz, bg and regions by one logit);
  * four mask selections (XYZ_LOSS_MASK_GT, MASK_LOSS_GT, REGION_LOSS_MASK_GT): the shipped visib / trunc / visib, all three
    different, one mask for all three (one pointer passed three times) and the mask-loss target shared with the region weight;
  * soft masks (0.3 / 0.7: BCE uses them as given, CE truncates them to class 0), BCE logits of +-40, exact CE ties z0 == z1,
    and B = 80, whose 80 x 4096 pixels take a second turn of the grid-stride loop on a 132-SM H100.

The original entry points are these with (L1, MO = 1, visib / trunc / visib); both give bit-identical sums, losses and gradient
planes.  Bounds as in tests/test_loss_kernels_gpu.py (derived there): TOL2 = 1e-5 of each channel group for two-plane outputs,
plus one unit roundoff of the 16-bit storage format for single-plane ones; pixel losses 2e-6.  The measured worst errors on an
H100 80GB HBM3 are recorded next to each bound."""
import pytest
import torch

from loss_ref_common import HW, NCH, REPORT, check, grad_scale, nan_planes, unit_roundoff  # noqa: E402 (tests/ is on sys.path)
from oracle import mask_oracle as M

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

TOL2 = 1e-5
MODES = {"L1": 0, "BCE": 1, "CE": 2}
SELECTIONS = [("visib", "trunc", "visib"), ("obj", "visib", "trunc"), ("trunc", "trunc", "trunc"), ("visib", "obj", "obj")]
CASES = [("base", 4), ("soft", 3), ("edges", 3), ("b80", 80)]
LOSSES = ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_region")


def tol_for(planes: int, fp32: float = TOL2) -> float:
    return fp32 if planes == 2 else unit_roundoff() + fp32


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


def _inputs(case: str, B: int, mlt: str) -> dict:
    mo = M.mask_channels(mlt)
    nv = 68 + mo
    g = torch.Generator(device="cuda").manual_seed(2000 + 31 * B + 7 * len(case) + MODES[mlt])
    dev = "cuda"
    z = torch.randn(B * HW, 72, device=dev, generator=g) * 2.0
    z[:, nv:] = float("nan")  # padding floats of a logit row are never read
    gt_xyz = torch.rand(B, 3, HW, device=dev, generator=g)
    obj = (torch.rand(B, HW, device=dev, generator=g) < 0.7).float()
    visib = obj * (torch.rand(B, HW, device=dev, generator=g) < 0.85).float()
    trunc = visib * (torch.rand(B, HW, device=dev, generator=g) < 0.9).float()
    if case == "soft":
        # weights and targets of 0.3 / 0.7: a lost factor of m, or a CE target rounded instead of truncated, shows
        vals = torch.tensor([0.0, 0.3, 0.7, 1.0], device=dev)
        obj, visib, trunc = (vals[torch.randint(0, 4, (B, HW), device=dev, generator=g)] for _ in range(3))
    labels = torch.randint(0, 65, (B, HW), device=dev, generator=g)
    coord2d = torch.rand(B, 2, HW, device=dev, generator=g) * 2 - 1
    extents = torch.rand(B, 3, device=dev, generator=g) * 0.25 + 0.05
    if case in ("edges", "b80"):
        zv = z.view(B, HW, 72)
        for j in range(3):
            zv[:, 0:400:4, mo + j] = gt_xyz[:, j, 0:400:4]  # masked xyz residual exactly 0
        zv[:, 1:400:4, 0] = trunc[:, 1:400:4]  # L1 mask residual exactly 0 against the trunc target
        sgn = torch.where(torch.rand(B, 200, device=dev, generator=g) < 0.5, -40.0, 40.0)
        zv[:, 400:600, 0] = sgn  # BCE logits of +-40: exp(-|z|) = 4e-18, sigmoid saturates
        zv[:, 600:800, 1] = zv[:, 600:800, 0]  # CE: exact ties z0 == z1 (for MO = 1 an ordinary xyz logit)
        zv[:, 800:900, mo + 3:nv] = 0.7  # region ties
        labels[:, :50] = 0
        labels[:, 50:100] = 64
    masks = dict(obj=obj.contiguous(), visib=visib.contiguous(), trunc=trunc.contiguous())
    return dict(B=B, mlt=mlt, mo=mo, z=z.contiguous(), gt_xyz=gt_xyz, masks=masks, labels=labels.contiguous(), coord2d=coord2d,
                extents=extents)


def _ptrs(d, sel):
    return tuple(d["masks"][k].data_ptr() for k in sel)  # the same selection passes the same pointer


def _ref_losses(z64, d, sel):
    """oracle.mask_oracle.pixel_losses on the float64 logits (pixel-major [B * 4096, 72] -> NCHW)."""
    B, nv = d["B"], 68 + d["mo"]
    head = z64[:, :nv].reshape(B, 64, 64, nv).permute(0, 3, 1, 2)
    m = {k: v.double().view(B, 64, 64) for k, v in d["masks"].items()}
    batch = dict(roi_xyz=d["gt_xyz"].double().view(B, 3, 64, 64), roi_mask_trunc=m["trunc"], roi_mask_visib=m["visib"],
                 roi_mask_obj=m["obj"], roi_region=d["labels"].view(B, 64, 64))
    return M.pixel_losses(head, batch, d["mlt"], sel)


def _glue_ref(z64, d, with_2d):
    import torch.nn.functional as F

    B, mo = d["B"], d["mo"]
    head = z64[:, :68 + mo].reshape(B, 64, 64, 68 + mo).permute(0, 3, 1, 2)
    parts = [(head[:, mo:mo + 3] - 0.5) * d["extents"].double().view(B, 3, 1, 1)]
    if with_2d:
        parts.append(d["coord2d"].double().view(B, 2, 64, 64))
    parts.append(F.softmax(head[:, mo + 4:], dim=1))
    return torch.cat(parts, 1).permute(0, 2, 3, 1).reshape(B * HW, -1)


def _sums(d, sel):
    sums = torch.full((7,), float("nan"), dtype=torch.float64, device="cuda")
    _C().gdrn_pixel_loss_fwd_ex(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), *_ptrs(d, sel), d["labels"].data_ptr(), sums.data_ptr(),
                                d["B"], HW, MODES[d["mlt"]], d["mo"], _stream())
    return sums


def _finalize(sums, B, ex=True):
    losses = torch.full((8,), float("nan"), device="cuda")
    vis_out = torch.full((2,), float("nan"), device="cuda")
    pose_sums = torch.zeros(4, dtype=torch.float64, device="cuda")
    vis = torch.zeros(B, 2, device="cuda")
    fn = _C().gdrn_loss_finalize_ex if ex else _C().gdrn_loss_finalize
    fn(sums.data_ptr(), pose_sums.data_ptr(), vis.data_ptr(), losses.data_ptr(), vis_out.data_ptr(), B, HW, 1, _stream())
    return losses


@pytest.mark.parametrize("sel", SELECTIONS, ids=lambda s: "-".join(s))
@pytest.mark.parametrize("mlt", list(MODES))
@pytest.mark.parametrize("case,B", CASES)
def test_pixel_loss_fwd_ex_and_finalize(case, B, mlt, sel):
    d = _inputs(case, B, mlt)
    sums = _sums(d, sel)
    losses = _finalize(sums, B)
    torch.cuda.synchronize()
    L = _ref_losses(d["z"].double(), d, sel)
    m_xyz, m_reg = d["masks"][sel[0]].double(), d["masks"][sel[2]].double()
    # sums of 0 / 1 masks are exact integers; 0.3 / 0.7 masks round in the fp32 partials.  Measured: <= 7.2e-9
    check(f"mask sum_xyz[{case},{mlt}]", sums[5:6], m_xyz.sum().view(1), 1e-7)
    check(f"mask sum_region[{case},{mlt}]", sums[6:7], m_reg.sum().view(1), 1e-7)
    # per pixel a few fp32 roundings (|z m - gt m|, the stable BCE, logsumexp - z_label), then fp32 partial sums and fp64
    # atomics, as in test_loss_kernels_gpu.py: 2e-6 of each loss.  Measured: <= 7.2e-8 (region), mask loss 5.5e-8
    tag = f"[{case},{mlt},{'-'.join(sel)}]"
    for i, k in enumerate(LOSSES):
        check(f"mask pixel {k}{tag}", losses[i:i + 1], L[k].view(1), 2e-6)


def _din(B, planes, seed):
    from gdr_net_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * HW, 128, device="cuda", generator=g) * (5e-4 * grad_scale())
    return ops.PT.from_float(x, planes)


@pytest.mark.parametrize("with_2d,planes", [(1, 2), (0, 1)])
@pytest.mark.parametrize("sel", SELECTIONS, ids=lambda s: "-".join(s))
@pytest.mark.parametrize("mlt", list(MODES))
@pytest.mark.parametrize("case,B", CASES)
def test_head_bwd_ex(case, B, mlt, sel, with_2d, planes):
    """d/d logits of sum_i gw_i L_i + <din, glue(logits)> with no din, a one-plane din and a two-plane din."""
    d = _inputs(case, B, mlt)
    mo, nv = d["mo"], 68 + d["mo"]
    sums = _sums(d, sel)
    gw = torch.tensor([0.7, -1.3, 2.1, 0.4, 1.7, 1.0, 1.0, 1.0], device="cuda") * grad_scale()
    nch = NCH[with_2d]
    for dmode in (None, 1, 2):
        din = _din(B, dmode, 11 + B) if dmode else None
        out = nan_planes((B * HW, 128), planes)
        _C().gdrn_head_bwd_ex(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), *_ptrs(d, sel), d["labels"].data_ptr(), sums.data_ptr(),
                              gw.data_ptr(), din.hi_ptr if din else None, din.lo_ptr if din else None, d["extents"].data_ptr(),
                              out.hi_ptr, out.lo_ptr, B, HW, with_2d, MODES[mlt], mo, _stream())
        torch.cuda.synchronize()
        z = d["z"].double().requires_grad_(True)
        L = _ref_losses(z, d, sel)
        tot = sum(float(gw[i]) * L[k] for i, k in enumerate(LOSSES))
        if din is not None:
            tot = tot + (din.float().double()[:, :nch] * _glue_ref(z, d, with_2d)).sum()
        (ref,) = torch.autograd.grad(tot, z)
        got = out.float()
        tag = f"[{case},{mlt},{'-'.join(sel)},{with_2d},din{dmode},{planes}]"
        # measured: planes 2 <= 1.9e-6 (regions, where the softmax backward subtracts), mask 2.8e-7, bg 7.3e-7, xyz 1.5e-7;
        # planes 1 <= 4.7e-4 (u of fp16 = 4.9e-4)
        tol = tol_for(planes)
        check(f"mask head_bwd mask{tag}", got[:, :mo], ref[:, :mo], tol)
        check(f"mask head_bwd xyz{tag}", got[:, mo:mo + 3], ref[:, mo:mo + 3], tol)
        check(f"mask head_bwd bg{tag}", got[:, mo + 3], ref[:, mo + 3], tol)
        check(f"mask head_bwd regions{tag}", got[:, mo + 4:nv], ref[:, mo + 4:nv], tol)
        pad = out.buf[:, :, nv:]
        assert bool((pad == 0).all()), ("columns >= 68 + MO not exactly zero", int((pad != 0).sum()))


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("with_2d", [1, 0])
@pytest.mark.parametrize("mlt", ["L1", "CE"])
def test_head_glue_fwd_ex(mlt, with_2d, planes):
    d = _inputs("edges", 3, mlt)
    out = nan_planes((3 * HW, 128), planes)
    _C().gdrn_head_glue_fwd_ex(d["z"].data_ptr(), d["coord2d"].data_ptr() if with_2d else None, d["extents"].data_ptr(), out.hi_ptr,
                               out.lo_ptr, 3, HW, with_2d, d["mo"], _stream())
    torch.cuda.synchronize()
    ref = _glue_ref(d["z"].double(), d, with_2d)
    nch = NCH[with_2d]
    check(f"mask glue[{mlt},{with_2d},{planes}]", out.float()[:, :nch], ref, tol_for(planes))  # measured: 2.4e-7 / 3.9e-4
    assert bool((out.buf[:, :, nch:] == 0).all())


@pytest.mark.parametrize("case,B", CASES)
def test_original_entry_points_equal_ex_defaults(case, B):
    """gdrn_pixel_loss_fwd / head_bwd / head_glue_fwd / loss_finalize == the _ex entry points with (L1, MO = 1, visib, trunc,
    visib), bit for bit; the six-slot sums buffer of the original ones is not written past slot 5."""
    d = _inputs(case, B, "L1")
    C = _C()
    old = torch.full((8,), float("nan"), dtype=torch.float64, device="cuda")
    m = d["masks"]
    C.gdrn_pixel_loss_fwd(d["z"].data_ptr(), d["gt_xyz"].data_ptr(), m["visib"].data_ptr(), m["trunc"].data_ptr(), d["labels"].data_ptr(),
                          old.data_ptr(), B, HW, _stream())
    new = _sums(d, ("visib", "trunc", "visib"))
    torch.cuda.synchronize()
    assert torch.equal(old[:6], new[:6]) and bool(old[6:].isnan().all()), (old, new)
    assert torch.equal(new[6], new[5])
    assert torch.equal(_finalize(old[:6].clone(), B, ex=False), _finalize(new, B, ex=True))
    gw = torch.tensor([0.7, -1.3, 2.1, 0.4, 1.7, 1.0, 1.0, 1.0], device="cuda") * grad_scale()
    for with_2d in (1, 0):
        for dmode in (None, 1, 2):
            din = _din(B, dmode, 5) if dmode else None
            outs = []
            for ex in (False, True):
                out = nan_planes((B * HW, 128), 2)
                args = (d["z"].data_ptr(), d["gt_xyz"].data_ptr())
                tail = (d["labels"].data_ptr(), (new if ex else old).data_ptr(), gw.data_ptr(), din.hi_ptr if din else None,
                        din.lo_ptr if din else None, d["extents"].data_ptr(), out.hi_ptr, out.lo_ptr, B, HW, with_2d)
                if ex:
                    C.gdrn_head_bwd_ex(*args, *_ptrs(d, ("visib", "trunc", "visib")), *tail, 0, 1, _stream())
                else:
                    C.gdrn_head_bwd(*args, m["visib"].data_ptr(), m["trunc"].data_ptr(), *tail, _stream())
                outs.append(out)
            torch.cuda.synchronize()
            assert torch.equal(outs[0].buf, outs[1].buf), (with_2d, dmode)
        outs = []
        for ex in (False, True):
            out = nan_planes((B * HW, 128), 2)
            a = (d["z"].data_ptr(), d["coord2d"].data_ptr() if with_2d else None, d["extents"].data_ptr(), out.hi_ptr, out.lo_ptr, B, HW,
                 with_2d)
            C.gdrn_head_glue_fwd_ex(*a, 1, _stream()) if ex else C.gdrn_head_glue_fwd(*a, _stream())
            outs.append(out)
        torch.cuda.synchronize()
        assert torch.equal(outs[0].buf, outs[1].buf)
