"""gdr_net_b200 -- H100-native (sm_90a) implementation of the GDR-Net train/infer hot path.

Public surface mirrors the reference module `core.gdrn_modeling.models.GDRN`:

    from gdr_net_b200 import GDRN
    model, optimizer = GDRN.build_model_optimizer(cfg)      # cfg: mmcv-style config (see gdr_net_b200.config)
    out_dict, loss_dict = model(roi_img, gt_xyz=..., ..., do_loss=True)

All math runs in hand-written CUDA kernels behind the C ABI declared in include/gdrn_b200.h.
"""
__version__ = "0.1.0"
