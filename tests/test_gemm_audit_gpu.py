"""GPU: every GEMM launch of a real engine step, audited against float64 (tests/gemm_audit.py).

The engine runs eagerly on one stream on the benchmark's workload (seeded weights, synth.make_batch(64, seed=100)), and
each launch of gemm_fwd_kernel / gemm_wgrad_kernel is compared element by element with a float64 reference built from that
launch's own operands.  At B = 64 almost every launch gives a persistent CTA 2..60 tiles, on the 128-wide tiles that do
most of the work: the shapes the synthetic op tests (tests/test_ops_gpu.py, tests/test_engine_ops_gpu.py) do not reach.
The single-pass "half" mode runs the same B = 64 step and the stand-alone Patch-PnP at the benchmark's B = 512: its
large plain-epilogue forwards (the stride-2 convs among them) are the launches of the 256-row tile, and its epilogue
statistics and folded epilogues are the nsplit-1 variants of the mixed mode's.  test_coverage_b64 asserts that the audit
reached what it was written for."""
import time

import pytest
import torch

import gemm_audit as GA  # noqa: E402 (tests/ is on sys.path: rootdir conftest)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    GA.print_report()


def _engine(precision, B):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200 import synth
    from gdr_net_b200.config import a6_config
    from oracle import fixtures

    sd = synth.seeded_state_dict(fixtures.template_from_manifest(), 0)
    model, _ = G.build_model_optimizer(a6_config(device="cuda"), precision=precision)
    model.load_state_dict(sd)
    model.train()
    b = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in synth.make_batch(B, seed=100).items()}
    aux = dict(roi_coord_2d=b["roi_coord_2d"], roi_cams=b["roi_cam"], roi_centers=b["roi_center"], roi_whs=b["roi_wh"],
               roi_extents=b["roi_extent"], resize_ratios=b["resize_ratio"], gt_xyz=b["roi_xyz"], gt_mask_trunc=b["roi_mask_trunc"],
               gt_mask_visib=b["roi_mask_visib"], gt_region=b["roi_region"], gt_ego_rot=b["ego_rot"], gt_points=b["roi_points"],
               sym_infos=None, gt_trans=b["trans"], gt_trans_ratio=b["roi_trans_ratio"])
    aux = {k: (v.float().contiguous() if isinstance(v, torch.Tensor) and v.dtype != torch.long else v) for k, v in aux.items()}
    eng = model.engine
    eng.wgrad_side_stream = False  # one stream: each wrapper reads its launch's result right after it
    return model, eng, b["roi_img"].float().contiguous(), aux


def _label(eng):
    def label(wp):
        tables = [("wf", eng.wf), ("wd", eng.wd), ("folded", getattr(eng, "_fold", None) and eng._fold["wf"] or {})]
        for tname, tab in tables:
            for key, t in tab.items():
                if t.buf.data_ptr() == wp.buf.data_ptr():
                    return f"{tname}[{key}]"
        return "?"

    return label


def _patch_pnp(precision, B, nIn=69):
    """The stand-alone Patch-PnP of the benchmark (seeded weights and maps), eagerly: () -> runs one forward, and its label."""
    from gdr_net_b200 import ops, synth
    from gdr_net_b200.GDRN import ConvPnPNet
    from gdr_net_b200.patch_pnp import PatchPnP

    net = ConvPnPNet(nIn=nIn).cuda()
    sd = synth.seeded_state_dict({"pnp_net." + k: v for k, v in net.state_dict().items()}, seed=11)
    net.load_state_dict({k[len("pnp_net."):]: v for k, v in sd.items()})
    net.eval()
    g = synth._gen(7, "pnp_bench")
    coor = torch.rand(B, nIn - 64, 64, 64, generator=g).cuda()
    region = torch.softmax(2.0 * torch.randn(B, 64, 64, 64, generator=g), dim=1).cuda()
    ext = (0.05 + 0.25 * torch.rand(B, 3, generator=g)).cuda()
    runner = PatchPnP(net, precision)
    runner.use_cuda_graphs = False  # eager: each wrapper reads its launch's result right after it
    runner(coor, region, ext)  # packs the weights, so that the label can name them
    torch.cuda.synchronize()

    def label(wp):  # (wf also holds the fp32 w_rt / b_rt the fc_rt operand is packed from)
        return next((f"wf[{k}]" for k, t in runner.wf.items() if isinstance(t, ops.PT) and t.buf.data_ptr() == wp.buf.data_ptr()), "?")

    return (lambda: runner(coor, region, ext)), label


RUNS = {}  # name -> (records, launches seen at the C ABI, seconds) or the exception of a failed audit (never re-run)


def _run(name, precision="mixed", B=64, mode="train"):
    if name not in RUNS:
        if mode == "patch_pnp":
            step, label = _patch_pnp(precision, B)
        else:
            model, eng, x, aux = _engine(precision, B)
            if mode == "eval":  # move the running statistics off their initial (0, 1), so the folded row scales differ per channel
                eng.forward(x[:4].contiguous(), {k: (v[:4].contiguous() if isinstance(v, torch.Tensor) else v) for k, v in aux.items()},
                            train_bn=True, do_loss=False)
            label = _label(eng)

            def step():
                if mode == "train":
                    eng.forward(x, aux, train_bn=True, do_loss=True)
                    eng.backward(torch.ones(8, device="cuda"))
                elif mode == "atomic_stats":
                    eng.deterministic = False  # BatchNorm statistics accumulated in the GEMM epilogue
                    eng.forward(x, aux, train_bn=True, do_loss=False)
                else:
                    model.eval()
                    eng.forward_eval_folded(x, aux)
        torch.cuda.synchronize()
        t0 = time.time()
        try:
            with GA.Audit(label=label) as au:
                step()
                torch.cuda.synchronize()
            RUNS[name] = (au.records, au.c_launches, time.time() - t0)
            print(f"{name}: {au.n_audited()} launches audited in {RUNS[name][2]:.1f} s")
        except Exception as e:  # noqa: BLE001 (kept, so that the coverage test reports it instead of repeating the launch)
            RUNS[name] = e
        del step, label
        torch.cuda.empty_cache()
    if isinstance(RUNS[name], Exception):
        raise RUNS[name]
    records, c_launches, _ = RUNS[name]
    audited = sum(1 for r in records if r["op"] != "unpack_wgrad")
    assert audited == c_launches, f"{name}: {c_launches} GEMM launches reached the library, {audited} passed the audit wrappers"
    return records


B64 = dict(mixed_train=dict(), fp32x3_train=dict(precision="fp32x3"), mixed_atomic_stats=dict(mode="atomic_stats"),
           mixed_eval_folded=dict(mode="eval"), half_train=dict(precision="half"),
           half_atomic_stats=dict(precision="half", mode="atomic_stats"), half_eval_folded=dict(precision="half", mode="eval"))
PNP512 = dict(precision="half", B=512, mode="patch_pnp")  # the benchmark's stand-alone Patch-PnP (nIn = 69)


@pytest.mark.parametrize("name", list(B64))
def test_audit_b64(name):
    """mixed train: 3-pass forward <128,3> / <64,3>, single-pass dgrad <128,1> / <64,1>, the phase dgrad, weight gradients
    <256,1> <192,1> <128,1> <64,1>, the fp32 logits with bias and ldc 72, the FC stack, the stem GEMM.  fp32x3 train: 3-pass
    dgrad and weight gradients <128,3> <64,3>.  atomic statistics: the BatchNorm sums of the epilogue over many tiles per
    CTA, incl. the deconvolution forward (4 phases) and the stem.  folded eval: bias + residual + ReLU on 128-wide tiles over
    row-scaled weights.  half: the same steps single-pass; the large plain-epilogue forwards on 256-row tiles <128,1>, the
    epilogue statistics and the folded bias / residual epilogues at nsplit 1."""
    records = _run(name, **B64[name])
    ops_seen = {r["op"] for r in records}
    if name.endswith("train"):
        assert ops_seen == set(GA.Audit.OPS), ops_seen
    else:
        assert {"conv_fwd", "gemm_fwd", "conv_dgrad_s2"} <= ops_seen, ops_seen


def test_audit_patch_pnp_b512():
    """Half Patch-PnP at B = 512: the three 3x3 s2 convs on 256-row tiles (64^2 -> 32^2 over the 69 -> 128 padded input,
    32^2 -> 16^2, and 16^2 -> 8^2 with two images per 128-row A box), then fc1 / fc2 / fc_rt."""
    records = _run("half_patch_pnp_b512", **PNP512)
    convs = [r for r in records if r["op"] == "conv_fwd"]
    assert len(convs) == 3 and all(r["stride"] == 2 and r["KH"] == 3 for r in convs), [r["name"] for r in convs]


@pytest.mark.parametrize("B", [3, 20])
def test_audit_small_batches(B):
    """B = 3: the 8 x 8 layers pack two images per 128-row tile, so the last tile is half empty; every weight gradient picks
    its K-split from kb_total / 8.  B = 20: layer3 (4 * B = 80 wide tiles) takes the third branch of pick_block_n, between
    half a wave and 0.75 waves."""
    records = _run(f"mixed_train_b{B}", B=B)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if B == 20 and sms == 132:
        l3 = [r for r in records if r["op"] == "conv_fwd" and r["groups"] == 80 and r["variant"] // 10 == 128]
        assert l3, "no launch in the middle branch of pick_block_n"
    if B == 3:
        assert any(r["op"] == "conv_wgrad" and r["ksplit"] > 1 for r in records)


def test_coverage_b64():
    """What the B = 64 audits must have reached; computed from the shapes, the variant's width and the SM count."""
    fwd, wg, runs = [], [], dict(B64, half_patch_pnp_b512=PNP512)
    for name, kw in runs.items():
        recs = _run(name, **kw)
        fwd += [dict(r, run=name) for r in recs if r["op"] in ("conv_fwd", "gemm_fwd", "conv_dgrad_s2")]
        wg += [r for r in recs if r["op"] in ("conv_wgrad", "gemm_wgrad")]
    assert {r["variant"] for r in fwd} == {1283, 643, 1281, 641}
    for v in (1283, 643, 1281, 641):
        multi = [r for r in fwd if r["variant"] == v and r["max_per_cta"] > 1 and r["remainder"] != 0]
        assert multi, f"no <{v // 10},{v % 10}> launch with several tiles per CTA and a remainder"
    assert any(r["nphase"] == 4 and r["max_per_cta"] > 1 for r in fwd), "no phase dgrad with several groups per CTA"
    assert any(r["stats"] and r["max_per_cta"] > 1 for r in fwd), "no epilogue statistics over several tiles per CTA"
    assert any(r["stats"] and r["nphase"] == 4 for r in fwd), "the deconvolution forward with epilogue statistics"
    assert {(r["width"], r["nsplit"]) for r in wg} == {(256, 1), (192, 1), (128, 1), (64, 1), (128, 3), (64, 3)}
    assert any(r["ksplit"] > 1 for r in wg)
    # the 256-row tile (at 132 SMs: ceil(M / 256) * n-tiles >= 99).  Mixed reaches it only with the stride-1 dgrads; the half
    # forward adds layer2.0.conv1 (3x3 s2, 256 tall tiles on 132 CTAs), the layer2.0 / layer3.0 1x1 s2 downsamples and
    # Patch-PnP features.6 at B = 512 (8^2 outputs: 128 tall tiles of 4 images)
    tall = [r for r in fwd if r["block_m"] == 256]
    assert {r["variant"] for r in tall} == {1281} and {r["block_m"] for r in fwd if r["variant"] == 1281} == {128, 256}
    for k in (3, 1):
        assert any(r["stride"] == 2 and r["KH"] == k for r in tall), f"no tall {k}x{k} stride-2 conv"
    assert any(r["TN"] == 2 for r in tall), "no tall launch with two images per 128-row box"
    assert any(r["max_per_cta"] > 1 and r["remainder"] != 0 for r in tall), "no tall launch with several tiles per CTA and a remainder"
    assert any(r["stats"] and r["variant"] % 10 == 1 and r["max_per_cta"] > 1 for r in fwd), "no nsplit-1 epilogue statistics over several tiles per CTA"
    assert any(r["run"] == "half_eval_folded" and r["bias"] for r in tall), "no folded tall launch with bias"
    secs = {n: round(RUNS[n][2], 1) for n in runs}
    print("audit wall time per run (s):", secs)


# ------------------------------------------------------------------------------------------------ packed operands
def _close(got, want, planes, what):
    """A packed operand decoded back against its fp32 parameter: one 16-bit rounding (planes 1) or the 2^-22 two-plane
    split (planes 2), plus the fp32 rounding of a folded row scale."""
    from gdr_net_b200 import ops

    fi = torch.finfo(ops.storage_format()[0])
    rel = (fi.eps / 2 if planes == 1 else 2.0 ** -22) + 2.0 ** -23
    bad = (got - want.double()).abs() > rel * want.double().abs() + fi.smallest_normal * fi.eps
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements differ from the parameter"


def test_packed_operands_decode_to_parameters():
    """eng.wf / eng.wd after prepare_weights(True) and the folded table after prepare_weights_folded(): the batched pack (one
    launch over a job table, with a per-row scale for the folded operands) against the parameters themselves."""
    model, eng, x, aux = _engine("mixed", 4)
    eng.forward(x, aux, train_bn=True, do_loss=False)  # running statistics away from (0, 1)
    model.eval()
    eng.prepare_weights(True)
    fold = eng.prepare_weights_folded()
    torch.cuda.synchronize()
    m = model
    convs = dict(eng._conv_modules())
    n = 0
    for key, conv in convs.items():
        O, I, k, _ = conv.weight.shape
        _close(GA.decode_conv_fwd(GA.pt64(eng.wf[key]), O, I, k, k), conv.weight, eng.planes, f"wf[{key}]")
        _close(GA.decode_conv_dgrad(GA.pt64(eng.wd[key]), O, I, k, k), conv.weight, eng.bplanes, f"wd[{key}]")
        n += 2
    assert eng.wd["rot_head_net.features.23"].shape == (256, 128)
    dc = m.rot_head_net.features[0].weight  # ConvTranspose2d IOHW [512][256][3][3]
    _close(GA.decode_conv_dgrad(GA.pt64(eng.wf["deconv"]), 512, 256, 3, 3), dc, eng.planes, "wf[deconv]")
    _close(GA.decode_deconv_dgrad(GA.pt64(eng.wd["deconv"]), 512, 256, 3, 3), dc, eng.bplanes, "wd[deconv]")
    _close(GA.decode_stem(GA.pt64(eng.wf["stem"])), m.backbone.conv1.weight, eng.planes, "wf[stem]")
    pn = m.pnp_net
    w_rt = torch.cat([pn.fc_r.weight, pn.fc_t.weight], 0)
    for key, w, nf in (("fc1", pn.fc1.weight, (128, 8, 8)), ("fc2", pn.fc2.weight, None), ("fc_rt", w_rt, None)):
        N, K = w.shape
        _close(GA.decode_linear(GA.pt64(eng.wf[key]), N, K, nhwc_from=nf), w, eng.planes, f"wf[{key}]")
        _close(GA.decode_linear(GA.pt64(eng.wd[key]), N, K, nhwc_from=nf, transpose=True), w, eng.bplanes, f"wd[{key}]")
    spread = 0.0
    for ck, bk in eng._conv_bn_pairs():
        bn = eng._bn_mods[bk]
        scale = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
        _close(fold["scale"][bk].double(), scale, 2, f"folded scale[{bk}]")
        _close(fold["shift"][bk].double(), bn.bias.double() - bn.running_mean.double() * scale, 2, f"folded shift[{bk}]")
        sc = fold["scale"][bk].double().view(-1, 1, 1, 1)  # the kernel multiplies by the fp32 scale it folded
        p = GA.pt64(fold["wf"][ck])
        if ck == "stem":
            got, want = GA.decode_stem(p), m.backbone.conv1.weight.double() * sc
        elif ck == "deconv":  # rows of the packed operand = output channels = dim 1 of the IOHW weight
            got, want = GA.decode_conv_dgrad(p, 512, 256, 3, 3), dc.double() * sc.view(1, -1, 1, 1)
        else:
            O, I, k, _ = convs[ck].weight.shape
            got, want = GA.decode_conv_fwd(p, O, I, k, k), convs[ck].weight.double() * sc
        _close(got, want, eng.planes, f"folded[{ck}]")
        spread = max(spread, float((scale.abs().max() / scale.abs().min()).detach()))
    assert spread > 1.05, "the folded row scales are all alike: the check would not see a missing scale"
