"""TEST INFRASTRUCTURE ONLY -- golden vectors for DropBlock on the Patch-PnP input (PNP_NET.PNP_HEAD_CFG.drop_prob /
dropblock_size), produced by the UNMODIFIED reference model (GDRN.py, conv_pnp_net.py, core/utils/dropblock) built from the a6
config with only these switches changed (the GPU box has no reference install).  torch.rand is wrapped during the forward to
record the uniform draw of DropBlock2D; the seed mask is that draw compared with the reference's own gamma.  The schedule
position is set through the reference's `pnp_net.dropblock.i`:

  ship_b5       the shipped head (64 regions, attention, 2-D coordinates), drop_prob 0.25, block 5, step 4999 (p = 0.25)
  r8_b3         8 regions with attention, drop_prob 0.5, block 3, step 2500 (mid-schedule)
  r32_noatt_b4  32 regions without attention, drop_prob 0.25, block 4 (the even crop), step 4200
  eval          the shipped head, drop_prob 0.25, block 5, step 4999, one eval forward: equal to the model without DropBlock

Each train case: a seeded batch of four crops, the losses, a few parameter gradients after `sum(loss_dict.values()).backward()`
and the seed mask.  Output: tests/golden/train_dropblock_b4.npz, keys "<case>/loss/<name>", "<case>/grad/<param>",
"<case>/seeds" (uint8 [4, 64, 64]), "<case>/step", "eval/{rot,trans}" and "eval/{rot,trans}_nodb".
Usage: python -m oracle.make_golden_dropblock"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200 import synth  # noqa: E402
from gdr_net_b200.config import Config, postprocess_like_main_gdrn  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden import REF_CFG  # noqa: E402

# name -> (ROT_HEAD switches, PNP_NET switches, drop_prob, dropblock_size, step, weight seed, batch seed)
CASES = {
    "ship_b5": (dict(NUM_REGIONS=64), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 0.25, 5, 4999, 51, 61),
    "r8_b3": (dict(NUM_REGIONS=8), dict(REGION_ATTENTION=True, WITH_2D_COORD=True), 0.5, 3, 2500, 52, 62),
    "r32_noatt_b4": (dict(NUM_REGIONS=32), dict(REGION_ATTENTION=False, WITH_2D_COORD=True), 0.25, 4, 4200, 53, 63),
}
EVAL = ("ship_b5", 54, 64)  # the configuration, weight seed, batch seed of the eval case
GRAD_KEYS = ("pnp_net.features.0.weight", "pnp_net.fc_r.weight", "rot_head_net.features.23.weight",
             "rot_head_net.features.23.bias", "backbone.bn1.weight")


def case_config(name, base, drop_prob=None):
    rh, pn, p, k, *_ = CASES[name]
    cfg = copy.deepcopy(base)
    cfg.MODEL.CDPN.ROT_HEAD.update(rh)
    cfg.MODEL.CDPN.PNP_NET.update(pn)
    cfg.MODEL.CDPN.PNP_NET.PNP_HEAD_CFG.update(drop_prob=p if drop_prob is None else drop_prob, dropblock_size=k)
    return cfg


class RecordRand:
    """torch.rand, recording every tensor it returns."""

    def __init__(self):
        self.draws, self._rand = [], torch.rand

    def __enter__(self):
        def rand(*a, **k):
            r = self._rand(*a, **k)
            self.draws.append(r.clone())
            return r

        torch.rand = rand
        return self

    def __exit__(self, *exc):
        torch.rand = self._rand


def build(ref_gdrn, base, name, wseed, drop_prob=None):
    torch.manual_seed(0)
    model, _ = ref_gdrn.build_model_optimizer(case_config(name, base, drop_prob))
    sd = synth.seeded_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    return model


def run_case(ref_gdrn, base, name, save):
    rh, _pn, p, k, step, wseed, bseed = CASES[name]
    model = build(ref_gdrn, base, name, wseed)
    batch = synth.make_batch(4, seed=bseed, num_regions=rh["NUM_REGIONS"])
    model.train()
    model.pnp_net.dropblock.i = step
    with RecordRand() as rec:
        _, loss_dict = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=True))
    assert len(rec.draws) == 1 and tuple(rec.draws[0].shape) == (4, 64, 64), [tuple(d.shape) for d in rec.draws]
    db = model.pnp_net.dropblock.dropblock
    seeds = (rec.draws[0] < db._compute_gamma(None)).to(torch.uint8)  # DropBlock2D.forward's own comparison
    sum(loss_dict.values()).backward()
    for n, v in loss_dict.items():
        save[f"{name}/loss/{n}"] = np.array(float(v))
    grads = dict(model.named_parameters())
    for n in GRAD_KEYS:
        save[f"{name}/grad/{n}"] = grads[n].grad.detach().numpy()
    save[f"{name}/seeds"], save[f"{name}/step"] = seeds.numpy(), np.array(step)
    print(name, "p", db.drop_prob, "seeds", int(seeds.sum()), {n: round(float(v), 6) for n, v in loss_dict.items()})


def run_eval(ref_gdrn, base, save):
    name, wseed, bseed = EVAL
    batch = synth.make_batch(4, seed=bseed)
    for suffix, drop_prob in (("", None), ("_nodb", 0.0)):
        model = build(ref_gdrn, base, name, wseed, drop_prob)
        model.eval()
        model.pnp_net.dropblock.i = CASES[name][4]
        with torch.no_grad(), RecordRand() as rec:
            out = model(batch["roi_img"].clone(), **synth.forward_kwargs(batch, train=False))
        assert not rec.draws
        save[f"eval/rot{suffix}"], save[f"eval/trans{suffix}"] = np.asarray(out["rot"]), out["trans"].numpy()
    print("eval", np.abs(save["eval/rot"] - save["eval/rot_nodb"]).max(), np.abs(save["eval/trans"] - save["eval/trans_nodb"]).max())


def main():
    torch.set_num_threads(os.cpu_count())
    ref_gdrn = ref_shim.import_reference_gdrn()
    base = Config.fromfile(os.path.join(ref_shim.REFERENCE_ROOT, REF_CFG))
    base = postprocess_like_main_gdrn(base, device="cpu")
    base.MODEL.CDPN.BACKBONE.PRETRAINED = ""
    save = {}
    for name in CASES:
        run_case(ref_gdrn, base, name, save)
    run_eval(ref_gdrn, base, save)
    path = os.path.join(ROOT, "tests", "golden", "train_dropblock_b4.npz")
    np.savez_compressed(path, **save)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
