"""Stand-alone Patch-PnP: `ConvPnPNet.forward(coor_feat, region, extents)` of the reference
(core/gdrn_modeling/models/conv_pnp_net.py:111-157) on the sm_90a kernels -- BASELINE.json configs[3]
("64x64x(3+64) correspondence maps -> R|t, batch 512").

    [B, 3|5, 64, 64] xyz (+2-D coords)  +  [B, R, 64, 64] region attention, if any  (+ extents [B, 3])
        -> gdrn_pnp_pack_input   NCHW fp32 -> NHWC 16-bit planes, nIn valid of round_up(nIn, 64) channels (64 or 128), xyz
                                 de-normalised; with drop_prob > 0 gdrn_dropblock_step first advances the DropBlock schedule and
                                 in train mode gdrn_pnp_pack_input_db multiplies the input by the block mask and its scale
        -> 3 x (wgmma implicit-GEMM conv 3x3 s2 -> GroupNorm(32)+ReLU)        64 -> 32 -> 16 -> 8
        -> fc1 (8192 -> 1024, LeakyReLU 0.1) -> fc2 (1024 -> 256, LeakyReLU) -> fc_r | fc_t (one 9-column GEMM)
        -> rot [B, 6], t [B, 3]  (fp32)

Inference only (no autograd): inside `GDRN.forward` the same kernels run with saved activations and a hand-written
backward (engine.py).  The whole sequence is replayed as ONE CUDA graph per batch shape.  There is no CPU fallback.
"""
from __future__ import annotations

import torch

from . import ops
from .capi import C
from .ops import PT, _stream


def dropblock_step(net, B: int, train: bool, dev):
    """One forward of `net`'s DropBlock schedule (a ConvPnPNet with drop_prob > 0, conv_pnp_net.py:128-142): gdrn_dropblock_step
    advances the device-resident counter and, in train mode, samples the block mask of B 64 x 64 crops.  Returns the device
    (keep [B*4096] uint8, scale [1] fp32) of that mask in train mode, else None.  The buffers of a batch size are allocated
    once, so captured graphs keep valid addresses; net.dropblock_seeds / dropblock_keep / dropblock_scale view them."""
    step = net.dropblock_counter(dev)
    if not train:
        C.gdrn_dropblock_step(step.data_ptr(), 0, 0, net.drop_prob, net.dropblock_size, 0, None, None, None, None, 0, 64, 64,
                              _stream())
        return None
    bufs = net._db_bufs.get(B)
    if bufs is None or bufs[0].device != step.device:
        bufs = net._db_bufs[B] = (torch.empty(B * 4096, dtype=torch.uint8, device=step.device),
                                  torch.empty(B * 4096, dtype=torch.uint8, device=step.device),
                                  torch.empty(B, dtype=torch.int32, device=step.device), torch.empty(1, device=step.device))
    keep, seeds, counts, scale = bufs
    seed = net.dropblock_seed & (2**64 - 1)
    C.gdrn_dropblock_step(step.data_ptr(), seed - 2**64 if seed >= 2**63 else seed, _rank(), net.drop_prob, net.dropblock_size, 1,
                          keep.data_ptr(), seeds.data_ptr(), counts.data_ptr(), scale.data_ptr(), B, 64, 64, _stream())
    net.dropblock_seeds, net.dropblock_keep, net.dropblock_scale = seeds.view(B, 64, 64), keep.view(B, 64, 64), scale
    return keep, scale


def _rank() -> int:
    import torch.distributed as dist

    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def pnp_net_forward(x: PT, net, wf: dict, b_rt: torch.Tensor, pred: torch.Tensor, saved: list | None = None):
    """3 x (conv 3x3 s2 -> GroupNorm + ReLU) -> fc1 -> fc2 -> fc_r|fc_t of `net` (a ConvPnPNet) on the input planes
    x [B, 64, 64, round_up(nIn, 64)].  wf: packed operands "pnp_net.features.{0,3,6}" (pack_conv_fwd), "fc1", "fc2" and "fc_rt"
    (pack_linear of fc_r and fc_t stacked), b_rt their stacked bias.  pred [B, 16] fp32 receives rot in its first
    fc_r.out_features columns and t in the next 3.  saved: receives dict(ci, gi, x_in, u, y, gstats) per conv for backward.
    Returns the inputs of fc1, fc2 and fc_r|fc_t."""
    B = x.shape[0]
    cur = x
    for ci, gi in ((0, 1), (3, 4), (6, 7)):
        gn = net.features[gi]
        u = ops.conv_fwd(cur, wf[f"pnp_net.features.{ci}"], 128, 3, 3, 2, 1)
        gstats = torch.empty(B, 32, 2, device=pred.device)
        y = ops.gn_relu_fwd(u, gn.weight, gn.bias, gstats, G=gn.num_groups, eps=gn.eps)
        if saved is not None:
            saved.append(dict(ci=ci, gi=gi, x_in=cur, u=u, y=y, gstats=gstats))
        cur = y
    flat = cur.view(B, 8192)
    h1 = ops.gemm_fwd(flat, wf["fc1"], 1024, bias=net.fc1.bias, act=1)
    h2 = ops.gemm_fwd(h1, wf["fc2"], 256, bias=net.fc2.bias, act=1)
    ops.gemm_fwd(h2, wf["fc_rt"], net.fc_r.out_features + 3, out_f32=pred, bias=b_rt, ldc=16, want_planes=False)
    return flat, h1, h2


class PatchPnP:
    def __init__(self, pnp_net, precision: str = "fp32x3"):
        precision = {"mixed": "fp32x3", "fp16": "half", "bf16": "half"}.get(precision, precision)
        assert precision in ("half", "fp32x3"), precision
        C.load()
        self.net = pnp_net
        self.planes = 1 if precision == "half" else 2
        self.precision = precision
        self.pnp_ld = -(-pnp_net.nIn // 64) * 64  # input row: 64 channels for nIn <= 64, else 128
        self.wf = {}
        self._wkey = None
        self._graphs = {}
        self.use_cuda_graphs = True

    # ------------------------------------------------------------------ weights (re-packed only when a parameter changed)
    def _prepare_weights(self):
        n = self.net
        key = tuple((p.data_ptr(), p._version) for p in n.parameters())
        if key == self._wkey:
            return
        pl, wf = self.planes, self.wf
        dev = n.fc1.weight.device
        for ci in (0, 3, 6):
            k = f"pnp_net.features.{ci}"
            wf[k] = ops.pack_conv_fwd(n.features[ci].weight.detach(), pl, out=wf.get(k), ipad=self.pnp_ld if ci == 0 else None)
        wf["fc1"] = ops.pack_linear(n.fc1.weight.detach(), pl, out=wf.get("fc1"), nhwc_from=(128, 8, 8))
        wf["fc2"] = ops.pack_linear(n.fc2.weight.detach(), pl, out=wf.get("fc2"))
        if "w_rt" not in wf:
            wf["w_rt"] = torch.empty(n.fc_r.out_features + 3, n.fc_r.in_features, device=dev)
            wf["b_rt"] = torch.empty(n.fc_r.out_features + 3, device=dev)
        with torch.no_grad():
            torch.cat([n.fc_r.weight, n.fc_t.weight], 0, out=wf["w_rt"])
            torch.cat([n.fc_r.bias, n.fc_t.bias], 0, out=wf["b_rt"])
        wf["fc_rt"] = ops.pack_linear(wf["w_rt"], pl, out=wf.get("fc_rt"))
        self._wkey = key
        self._graphs.clear()  # graphs hold the packed operands' addresses; buffers are reused, but stay safe

    # ------------------------------------------------------------------ the kernel sequence
    def _run(self, coor_feat, region, extents, pred, train: bool):
        B, c_feat = coor_feat.shape[0], coor_feat.shape[1]
        c_reg = 0 if region is None else region.shape[1]
        x = PT((B, 64, 64, self.pnp_ld), self.planes, device=coor_feat.device)
        args = (coor_feat.data_ptr(), c_feat, ops.ptr(region), c_reg, ops.ptr(extents), x.hi_ptr, x.lo_ptr, B, 4096)
        db = dropblock_step(self.net, B, train, coor_feat.device) if self.net.drop_prob > 0 else None
        if db is not None:
            C.gdrn_pnp_pack_input_db(*args, self.pnp_ld, db[0].data_ptr(), db[1].data_ptr(), _stream())
        elif self.pnp_ld == 128:
            C.gdrn_pnp_pack_input(*args, _stream())
        else:
            C.gdrn_pnp_pack_input_ex(*args, self.pnp_ld, _stream())
        pnp_net_forward(x, self.net, self.wf, self.wf["b_rt"], pred)

    @torch.no_grad()
    def __call__(self, coor_feat: torch.Tensor, region: torch.Tensor | None = None, extents: torch.Tensor | None = None,
                 train: bool = False):
        if not coor_feat.is_cuda:
            raise RuntimeError("gdr_net_b200 Patch-PnP runs on CUDA (sm_90a) only; there is no CPU fallback")
        n = self.net
        coor_feat = coor_feat.float().contiguous()
        region = None if region is None else region.float().contiguous()
        extents = None if extents is None else extents.float().contiguous()
        B, c_feat, H, W = coor_feat.shape
        c_reg = 0 if region is None else region.shape[1]
        if (H, W) != (64, 64) or c_feat + c_reg != n.nIn:
            raise ValueError(f"Patch-PnP expects [B, {n.nIn} = coor + region channels, 64, 64]; got {c_feat} + {c_reg} at {H}x{W}")
        if c_feat in (3, 5) and extents is None:
            raise ValueError("extents are required to de-normalise the xyz channels (conv_pnp_net.py:120-122)")
        self._prepare_weights()
        nr = n.fc_r.out_features
        if not self.use_cuda_graphs:
            pred = torch.zeros(B, 16, device=coor_feat.device)
            self._run(coor_feat, region, extents, pred, train)
            return pred[:, :nr].clone(), pred[:, nr:nr + 3].clone()
        key = (B, c_feat, c_reg, extents is not None, train)
        g = self._graphs.get(key)
        if g is None:
            st = dict(coor=coor_feat.clone(), region=None if region is None else region.clone(),
                      ext=None if extents is None else extents.clone(), pred=torch.zeros(B, 16, device=coor_feat.device))
            step = n.dropblock_counter(coor_feat.device).clone() if n.drop_prob > 0 else None
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._run(st["coor"], st["region"], st["ext"], st["pred"], train)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            if step is not None:  # the warm-up run does not count as a forward of the DropBlock schedule
                n.dropblock_counter(coor_feat.device).copy_(step)
            st["graph"] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(st["graph"]):
                self._run(st["coor"], st["region"], st["ext"], st["pred"], train)
            g = self._graphs[key] = st
        g["coor"].copy_(coor_feat, non_blocking=True)
        if region is not None:
            g["region"].copy_(region, non_blocking=True)
        if extents is not None:
            g["ext"].copy_(extents, non_blocking=True)
        g["graph"].replay()
        return g["pred"][:, :nr].clone(), g["pred"][:, nr:nr + 3].clone()
