"""TEST INFRASTRUCTURE ONLY -- golden copy of what the reference's own config files resolve to: `configs/gdrn/lm/a6_cPnP_lm13.py` (the
a6_cPnP LM model, solver learning rate and optimizer config after `_base_` merging and `_delete_`) and the YCB-V
`a6_cPnP_AugAAETrunc_BG0.5_Rsym_ycbv_real_pbr_visib20_10e.py` (symmetric PM loss), loaded from /root/reference with
`gdr_net_b200.config.Config.fromfile` and post-processed like main_gdrn.py.  Output: tests/golden/reference_configs.json.
Usage: python -m oracle.make_golden_configs"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gdr_net_b200.config import Config, postprocess_like_main_gdrn  # noqa: E402

REF = "/root/reference"


def main():
    ref = postprocess_like_main_gdrn(Config.fromfile(os.path.join(REF, "configs/gdrn/lm/a6_cPnP_lm13.py")), device="cpu")
    ycbv = Config.fromfile(os.path.join(REF, "configs/gdrn/ycbv/a6_cPnP_AugAAETrunc_BG0.5_Rsym_ycbv_real_pbr_visib20_10e.py"))
    cdpn = ref.MODEL.CDPN.to_dict()
    cdpn["BACKBONE"]["PRETRAINED"] = ""  # a download path in the reference; the model here starts from random weights
    gold = dict(lm13=dict(CDPN=cdpn, BASE_LR=ref.SOLVER.BASE_LR, OPTIMIZER_CFG=dict(ref.SOLVER.OPTIMIZER_CFG)),
                ycbv=dict(PM_LOSS_SYM=ycbv.MODEL.CDPN.PNP_NET.PM_LOSS_SYM))
    path = os.path.join(ROOT, "tests", "golden", "reference_configs.json")
    with open(path, "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
    print("wrote", path)


if __name__ == "__main__":
    main()
