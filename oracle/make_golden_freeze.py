"""TEST INFRASTRUCTURE ONLY -- golden vectors for the frozen sub-networks (MODEL.CDPN.BACKBONE.FREEZE, ROT_HEAD.FREEZE,
PNP_NET.FREEZE), produced by the UNMODIFIED reference (run in the build container; the GPU box has no /root/reference).

The reference model and optimizer are built from the a6 config with only the FREEZE switches changed, loaded with the calibrated
weights of oracle/fixtures.py (seed WSEED) and run in train mode on a seeded batch of four crops.  Per case (oracle/freeze_oracle.py
CASES: bb, head, pnp, bb_pnp, head_pnp, all) tests/golden/train_freeze_<case>_b4.npz holds:
  * loss/<name>        the loss dict;
  * none_grad          the names of the parameters whose .grad is None after sum(loss_dict.values()).backward();
  * grad/<name>        the gradients of GRAD_KEYS that belong to a live sub-network;
  * bn/<buffer>        the BN_KEYS running statistics and counters after the train-mode forward;
  * opt/lrs, opt/sizes the optimizer's param groups: learning rate and parameter count, in group order;
  * exc/build, exc/backward   the type name of the exception building the optimizer or running backward raised ("" if none).
With all three frozen the reference's optimizer gets an empty parameter list and building it raises; that case holds exc/build only.

Usage: python -m oracle.make_golden_freeze"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.config import Config, postprocess_like_main_gdrn  # noqa: E402
from oracle import fixtures, ref_shim  # noqa: E402
from oracle.freeze_oracle import CASES  # noqa: E402
from oracle.make_golden import REF_CFG  # noqa: E402

WSEED, BSEED = 3, 37
GRAD_KEYS = ("backbone.bn1.weight", "backbone.layer1.0.bn1.weight", "backbone.layer4.2.bn2.weight", "backbone.layer4.2.bn2.bias",
             "rot_head_net.features.1.weight", "rot_head_net.features.21.weight", "rot_head_net.features.23.weight",
             "rot_head_net.features.23.bias", "pnp_net.features.1.weight", "pnp_net.features.4.bias", "pnp_net.fc1.bias",
             "pnp_net.fc_r.weight")  # every small tensor: the files stay ~100 KB
BN_KEYS = [f"{m}.{b}" for m in ("backbone.bn1", "backbone.layer4.2.bn2", "rot_head_net.features.1", "rot_head_net.features.21")
           for b in ("running_mean", "running_var", "num_batches_tracked")]


def train_case(ref_gdrn, name):
    fb, fh, fp = CASES[name]
    cfg = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    cfg = postprocess_like_main_gdrn(cfg, device="cpu")
    cfg.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    cfg.MODEL.CDPN.BACKBONE.FREEZE, cfg.MODEL.CDPN.ROT_HEAD.FREEZE, cfg.MODEL.CDPN.PNP_NET.FREEZE = fb, fh, fp
    torch.manual_seed(0)
    save = {"exc/build": np.array(""), "exc/backward": np.array("")}
    try:
        model, optimizer = ref_gdrn.build_model_optimizer(copy.deepcopy(cfg))
    except Exception as e:  # all three frozen: no parameter left for the optimizer
        save["exc/build"] = np.array(type(e).__name__)
        print(name, "build raised", type(e).__name__, e)
        return _write(name, save)
    save["opt/lrs"] = np.array([g["lr"] for g in optimizer.param_groups], dtype=np.float64)
    save["opt/sizes"] = np.array([len(g["params"]) for g in optimizer.param_groups], dtype=np.int64)
    model.load_state_dict(fixtures.calibrated_state_dict(WSEED))
    batch = synth.make_batch(4, seed=BSEED)
    model.train()
    _, loss_dict = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=True))
    save.update({("loss/" + k): np.array(float(v)) for k, v in loss_dict.items()})
    bufs = dict(model.named_buffers())
    for k in BN_KEYS:
        save["bn/" + k] = bufs[k].detach().numpy().copy()
    try:
        sum(loss_dict.values()).backward()
    except Exception as e:  # nothing in the loss dict requires grad
        save["exc/backward"] = np.array(type(e).__name__)
        print(name, "backward raised", type(e).__name__, e)
    params = dict(model.named_parameters())
    save["none_grad"] = np.array([k for k, p in params.items() if p.grad is None])
    for k in GRAD_KEYS:
        if params[k].grad is not None:
            save["grad/" + k] = params[k].grad.detach().numpy()
    print(name, {k: float(v) for k, v in loss_dict.items()}, "groups", save["opt/sizes"].tolist(), save["opt/lrs"].tolist(),
          "None grads", len(save["none_grad"]))
    return _write(name, save)


def _write(name, save):
    path = os.path.join(ROOT, "tests", "golden", f"train_freeze_{name}_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    for name in CASES:
        train_case(ref_gdrn, name)


if __name__ == "__main__":
    main()
