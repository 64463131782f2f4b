"""GPU: every GEMM launch of a real engine step, audited against float64 (tests/gemm_audit.py).

The engine runs eagerly on one stream on the benchmark's workload (seeded weights, synth.make_batch(64, seed=100)), and
each launch of gemm_fwd_kernel / gemm_wgrad_kernel is compared element by element with a float64 reference built from that
launch's own operands.  At B = 64 almost every launch gives a persistent CTA 2..60 tiles, on the 128-wide tiles that do
most of the work: the shapes the synthetic op tests (tests/test_ops_gpu.py, tests/test_engine_ops_gpu.py) do not reach.
test_coverage_b64 asserts that the audit reached what it was written for."""
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


RUNS = {}  # name -> (records, launches seen at the C ABI, seconds) or the exception of a failed audit (never re-run)


def _run(name, precision="mixed", B=64, mode="train"):
    if name not in RUNS:
        model, eng, x, aux = _engine(precision, B)
        if mode == "eval":  # move the running statistics off their initial (0, 1), so the folded row scales differ per channel
            eng.forward(x[:4].contiguous(), {k: (v[:4].contiguous() if isinstance(v, torch.Tensor) else v) for k, v in aux.items()},
                        train_bn=True, do_loss=False)
        torch.cuda.synchronize()
        t0 = time.time()
        try:
            with GA.Audit(label=_label(eng)) as au:
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
            RUNS[name] = (au.records, au.c_launches, time.time() - t0)
            print(f"{name}: {au.n_audited()} launches audited in {RUNS[name][2]:.1f} s")
        except Exception as e:  # noqa: BLE001 (kept, so that the coverage test reports it instead of repeating the launch)
            RUNS[name] = e
        del model, eng, x, aux
        torch.cuda.empty_cache()
    if isinstance(RUNS[name], Exception):
        raise RUNS[name]
    records, c_launches, _ = RUNS[name]
    audited = sum(1 for r in records if r["op"] != "unpack_wgrad")
    assert audited == c_launches, f"{name}: {c_launches} GEMM launches reached the library, {audited} passed the audit wrappers"
    return records


B64 = dict(mixed_train=dict(), fp32x3_train=dict(precision="fp32x3"), mixed_atomic_stats=dict(mode="atomic_stats"),
           mixed_eval_folded=dict(mode="eval"))


@pytest.mark.parametrize("name", list(B64))
def test_audit_b64(name):
    """mixed train: 3-pass forward <128,3> / <64,3>, single-pass dgrad <128,1> / <64,1>, the phase dgrad, weight gradients
    <256,1> <192,1> <128,1> <64,1>, the fp32 logits with bias and ldc 72, the FC stack, the stem GEMM.  fp32x3 train: 3-pass
    dgrad and weight gradients <128,3> <64,3>.  atomic statistics: the BatchNorm sums of the epilogue over many tiles per
    CTA, incl. the deconvolution forward (4 phases) and the stem.  folded eval: bias + residual + ReLU on 128-wide tiles over
    row-scaled weights."""
    records = _run(name, **B64[name])
    ops_seen = {r["op"] for r in records}
    if name.endswith("train"):
        assert ops_seen == set(GA.Audit.OPS), ops_seen
    else:
        assert {"conv_fwd", "gemm_fwd", "conv_dgrad_s2"} <= ops_seen, ops_seen


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
    fwd, wg = [], []
    for name, kw in B64.items():
        recs = _run(name, **kw)
        fwd += [r for r in recs if r["op"] in ("conv_fwd", "gemm_fwd", "conv_dgrad_s2")]
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
    secs = {n: round(RUNS[n][2], 1) for n in B64}
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
