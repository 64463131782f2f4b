"""CPU: the geometry head's shape switches (ROT_HEAD.CONV_KERNEL_SIZE = 2 | 3 | 4, OUT_CONV_KERNEL_SIZE = 1 | 3).

  * the oracle restatement (oracle/head_shape_oracle.py) against the unmodified reference built with each head shape
    (tests/golden/train_head_shape_b4.npz, oracle/make_golden_head_shape.py): eval maps and pose, losses and every parameter gradient;
  * `build_model_optimizer` gives the reference's state_dict keys and shapes, parameter order and optimizer groups, and loads the
    reference-shaped weights with strict=True; every supported (k, k_out) pair builds; other kernel sizes, NUM_LAYERS and
    NUM_FILTERS are refused naming the key;
  * gdrn_conv_dgrad_s2 refuses (K, pad) pairs outside k3 p1 / k1 p0 / k4 p1 / k2 p0 without touching a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import gdrn_oracle as O
from oracle import head_shape_oracle as HS
from oracle.make_golden_head_shape import CASES, EVAL_STRIDE, grad_sample_index, make_batch
from oracle.make_golden_head_gn import read_json


def case_config(case, device="cpu", **kw):
    from gdr_net_b200.config import a6_config

    rh, pn, *_ = CASES[case]
    cfg = a6_config(device=device, **kw)
    for k, v in rh.items():
        setattr(cfg.MODEL.CDPN.ROT_HEAD, k, v)
    for k, v in pn.items():
        setattr(cfg.MODEL.CDPN.PNP_NET, k, v)
    return cfg


def oracle_kwargs(case):
    rh, pn, *_ = CASES[case]
    aware = dict(rot_aware=rh.get("ROT_CLASS_AWARE", False), mask_aware=rh.get("MASK_CLASS_AWARE", False),
                 region_aware=rh.get("REGION_CLASS_AWARE", False))
    return dict(k=rh["CONV_KERNEL_SIZE"], k_out=rh["OUT_CONV_KERNEL_SIZE"], G=rh["NUM_GN_GROUPS"] if rh.get("NORM") == "GN" else None,
                num_regions=rh["NUM_REGIONS"], mask_loss_type=rh.get("MASK_LOSS_TYPE", "L1"), region_att=pn["REGION_ATTENTION"],
                num_classes=rh.get("NUM_CLASSES", 1) if any(aware.values()) else 1, **aware)


def seeded_weights(case):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200 import synth

    model, _ = G.build_model_optimizer(case_config(case))
    return synth.seeded_state_dict(model.state_dict(), seed=CASES[case][3])


def golden(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "train_head_shape_b4.npz"))
    return {k[len(case) + 1:]: g[k] for k in g.files if k.startswith(case + "/")}


# ------------------------------------------------------------------------------------------------ oracle vs reference goldens
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    g = golden(golden_dir, case)
    sd = seeded_weights(case)
    batch = make_batch(case)
    kw = oracle_kwargs(case)
    with torch.no_grad():
        o = HS.gdrn_forward(O.leaf_state_dict(sd, requires_grad=False), batch, train=False, do_loss=False, **kw)
    assert np.abs(o["head"][:, :, ::EVAL_STRIDE, ::EVAL_STRIDE].numpy() - g["eval/head"]).max() <= 1e-5
    assert np.abs(o["trans"].numpy() - g["eval/trans"]).max() <= 1e-5
    assert np.abs(o["rot"].numpy() - g["eval/rot"]).max() <= 1e-5
    leaf = O.leaf_state_dict(sd)
    o = HS.gdrn_forward(leaf, batch, train=True, do_loss=True, update_stats=True, **kw)
    assert list(o["losses"]) == [k[len("loss/"):] for k in g if k.startswith("loss/")]
    for k, v in o["losses"].items():
        ref = float(g["loss/" + k])
        assert abs(float(v.detach()) - ref) <= 5e-6 * abs(ref), (k, float(v.detach()), ref)
    sum(o["losses"].values()).backward()
    names = [k[len("grad/"):] for k in g if k.startswith("grad/")]
    assert names == [n for n in sd if not n.endswith(("running_mean", "running_var", "num_batches_tracked"))]
    for name in names:
        ref = g["grad/" + name]
        mine = leaf[name].grad.reshape(-1).numpy()[grad_sample_index(leaf[name].numel())]
        err = np.abs(mine - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err <= 2e-5, (name, err)  # fp32 on the CPU: the backbone BatchNorm gradients sum 65536 pixels


# ------------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("case", list(CASES))
def test_build_surface_matches_the_reference(golden_dir, case):
    from gdr_net_b200 import GDRN as G

    g = golden(golden_dir, case)
    model, optimizer = G.build_model_optimizer(case_config(case))
    sd = model.state_dict()
    assert list(sd) == read_json(g["sd_keys"])
    assert [list(v.shape) for v in sd.values()] == read_json(g["sd_shapes"])
    names = {id(p): n for n, p in model.named_parameters()}
    groups = [dict(params=[names[id(p)] for p in grp["params"]], lr=grp["lr"]) for grp in optimizer.param_groups]
    assert groups == read_json(g["opt_groups"])
    assert model.load_state_dict(seeded_weights(case), strict=True) is not None
    rh = CASES[case][0]
    k, k_out = rh["CONV_KERNEL_SIZE"], rh["OUT_CONV_KERNEL_SIZE"]
    dc, oc = model.rot_head_net.features[0], model.rot_head_net.features[23]
    assert (dc.kernel_size, dc.stride, dc.padding, dc.output_padding) == ((k, k), (2, 2), (HS.DECONV_PADDING[k][0],) * 2,
                                                                          (HS.DECONV_PADDING[k][1],) * 2)
    assert (oc.kernel_size, oc.padding) == ((k_out, k_out), (k_out // 2, k_out // 2))


@pytest.mark.parametrize("k_out", [1, 3])
@pytest.mark.parametrize("k", [2, 3, 4])
def test_every_supported_shape_builds_and_keeps_64x64(k, k_out):
    from gdr_net_b200 import GDRN as G

    head = G.RotWithRegionHead(kernel_size=k, output_kernel_size=k_out)
    f = head.features
    assert f[0].weight.shape == (512, 256, k, k) and f[23].weight.shape == (69, 256, k_out, k_out)
    assert f[0].bias is None and f[23].bias is not None
    with torch.no_grad():
        y = f[0](torch.zeros(1, 512, 8, 8))
        assert y.shape == (1, 256, 16, 16)
        assert f[23](torch.zeros(1, 256, 64, 64)).shape == (1, 69, 64, 64)
    # the init of every shape: conv / deconv weights normal(0, 0.001), biases 0 (reference normal_init)
    for m in (f[0], f[23]):
        assert 0.0005 < float(m.weight.detach().std()) < 0.002 and float(m.weight.detach().mean().abs()) < 1e-3
    assert float(f[23].bias.abs().max()) == 0.0


@pytest.mark.parametrize("key,value", [("CONV_KERNEL_SIZE", 1), ("CONV_KERNEL_SIZE", 5), ("OUT_CONV_KERNEL_SIZE", 2),
                                       ("NUM_LAYERS", 2), ("NUM_FILTERS", 128)])
def test_unsupported_head_shape_rejected(key, value):
    from gdr_net_b200 import GDRN as G
    from gdr_net_b200.config import a6_config

    cfg = a6_config(device="cpu")
    setattr(cfg.MODEL.CDPN.ROT_HEAD, key, value)
    with pytest.raises(NotImplementedError) as e:
        G.build_model_optimizer(cfg)
    assert f"ROT_HEAD.{key} = {value}" in str(e.value)
    kw = dict(CONV_KERNEL_SIZE="kernel_size", OUT_CONV_KERNEL_SIZE="output_kernel_size", NUM_LAYERS="num_layers",
              NUM_FILTERS="num_filters")
    with pytest.raises(NotImplementedError) as e:
        G.RotWithRegionHead(**{kw[key]: value})
    assert f"ROT_HEAD.{key} = {value}" in str(e.value)


def test_conv_dgrad_s2_refuses_other_kernel_and_padding_pairs():
    from gdr_net_b200 import capi

    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("library not built")
    dll = capi.C.load()
    p = ctypes.c_void_p(16)  # never dereferenced: every call below fails its argument checks first
    for K, pad in ((5, 2), (4, 0), (2, 1), (3, 0), (1, 1), (6, 2)):
        assert dll.gdrn_conv_dgrad_s2(p, None, p, None, p, None, None, None, 4, 8, 8, 512, 256, 256, K, pad, 256, 0, 1, None) == -1
        assert f"got k{K} p{pad}".encode() in dll.gdrn_last_error(), dll.gdrn_last_error()
