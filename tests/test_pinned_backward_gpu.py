"""Every parameter gradient of a whole engine step, per output channel, against a float64 replay of the oracle that follows the
engine's own ReLU, max-pool and L1 decisions (tests/pinned_backward.py), on the bench.py workload.

What is left after pinning is backward arithmetic, so the bounds below are set by it, per channel: a wrong saved tensor or
bitmap handed to a backward launch, a weight gradient joined from the side stream too early, a loss scale removed from the wrong
segment, a wrong `unpack_wgrad` layout or bias column sum, or an fp16 activation gradient that underflows under the static loss
scale shows up in the channels it touches.  Each case also checks all 43 BatchNorm running means, variances and counters and a
per-layer forward parity of the engine's stored activations against the pinned float64 forward, and prints the worst channel
per tensor family and the decisions the float64 forward would have taken differently.

  mixed  B = 64   module API (`model(...)`, `.backward()`, `p.grad`): the bench.py path, fp16 backward at loss scale 1024
  fp32x3 B = 64   two-plane backward: a much tighter bound
  mixed  B = 64   `engine.deterministic = False`: epilogue statistics and atomic BatchNorm-backward sums
  mixed  B = 20   a batch that is not a power of two: other tails in every batch-sized loop
  mixed  B = 64   8 surface regions (ROT_HEAD.NUM_REGIONS = 8), replayed through oracle/region_oracle.py
"""
import gc

import pytest
import torch

import pinned_backward as PB
from gdr_net_b200 import synth
from gdr_net_b200.config import a6_config
from oracle import gdrn_oracle as O
from oracle import mask_oracle as M
from oracle import region_oracle as RO
from test_regions_cpu import CASES, oracle_kwargs, region_config  # noqa: E402 (tests/ is on sys.path)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

# Per-channel gradient bounds (e_r of tests/pinned_backward.py): (weight rows, entries of 1-D tensors).  Measured worst over the
# five cases on an H100 80GB HBM3 at 700 W:
#   fp32x3  rows 2.0e-3 (backbone.conv1.weight)   1-D 5.4e-3 (backbone.layer1.0.bn2.bias)
#   mixed   rows 1.4e-2 (r8: backbone.layer1.0.conv1.weight; 7.5e-3 .. 8.2e-3 in the shipped head, pnp_net.features.3.weight)
#           1-D 7.8e-2 (small entries of BatchNorm gamma / beta gradients whose tensors agree to 2e-3 rel-L2)
BOUND = {"fp32x3": (5e-3, 1.5e-2), "mixed": (4e-2, 2e-1)}
STAT_BOUND = 1e-4    # running mean / variance, in units of the step's update (momentum * batch std / variance); measured 1.4e-5
PARITY_BOUND = 1e-3  # rel-L2 of each stored activation against the pinned float64 forward; measured 7.9e-5 (rot_head_net.features.21)


@pytest.fixture(scope="module")
def workload():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import fixtures

    return synth.seeded_state_dict(fixtures.template_from_manifest(), 0)


def _shipped(precision, sd, B):
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(a6_config(device="cuda"), precision=precision)
    model.load_state_dict(sd)
    fwd = lambda leaf, b: O.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True)  # noqa: E731
    return model, sd, synth.make_batch(B, seed=100), fwd, (O,)


def _r8():
    from gdr_net_b200 import GDRN as G

    model, _ = G.build_model_optimizer(region_config("r8", device="cuda"), precision="mixed")
    sd = synth.seeded_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, seed=CASES["r8"][2])
    model.load_state_dict(sd)
    kw = oracle_kwargs("r8")
    fwd = lambda leaf, b: RO.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True, **kw)  # noqa: E731
    return model, sd, synth.make_batch(64, seed=100, num_regions=8), fwd, (O, M, RO)


CASE_IDS = ["mixed_b64", "fp32x3_b64", "mixed_b64_atomic", "mixed_b20", "r8_mixed_b64"]


@pytest.mark.parametrize("case", CASE_IDS)
def test_pinned_gradients(workload, case):
    if case == "r8_mixed_b64":
        model, sd, batch_cpu, fwd, modules = _r8()
    else:
        precision = "fp32x3" if case.startswith("fp32x3") else "mixed"
        model, sd, batch_cpu, fwd, modules = _shipped(precision, workload, 20 if case == "mixed_b20" else 64)
    precision = model.precision
    model.train()
    model.engine.deterministic = case != "mixed_b64_atomic"
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch_cpu.items()}
    for p in model.parameters():
        p.grad = None
    # the module API step, with the decisions taken between forward and backward (backward clears engine.saved)
    _, ld = model(batch["roi_img"], **synth.forward_kwargs(batch, train=True))
    pins = PB.capture(model.engine)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    params = dict(model.named_parameters())
    out, leaf, shim = PB.replay(fwd, sd, batch_cpu, pins, modules)
    del pins
    gc.collect()
    ref = {n: leaf[n].grad for n in params}
    fails, table = PB.compare_grads({n: p.grad for n, p in params.items()}, ref, *BOUND[precision])
    stats = PB.running_stat_errors(model, sd, leaf)

    tag = f"[{case}]"
    for k, v in ld.items():
        r = float(out["losses"][k].detach())
        print(f"{tag} {k}: engine {float(v.detach()):.6f} pinned float64 {r:.6f} rel {abs(float(v.detach()) - r) / abs(r):.1e}")
    for fam, (name, row, e, rel) in sorted(PB.worst_by_family(table).items()):
        print(f"{tag} worst e_r {fam:34s} {e:.2e}  ({name} row {row}, tensor rel-L2 {rel:.1e})")
    for one_d, what in ((False, "weight row"), (True, "1-D entry")):
        sub = [t for t in table if (ref[t[0]].dim() == 1) == one_d]
        worst = max(sub, key=lambda t: t[2] if t[2] == t[2] else float("inf"))
        print(f"{tag} WORST {what}: {worst[0]} row {worst[1]}: e_r {worst[2]:.3e} (bound {BOUND[precision][one_d]:.1e})")
    flips = {s["name"]: s["flips"] for s in shim.sites if s["flips"]}
    print(f"{tag} decision flips (float64 forward vs engine): {sum(flips.values())} of {sum(s['n'] for s in shim.sites)} "
          f"decisions, per site {flips}")
    par = max((s["parity"], s["name"]) for s in shim.sites if s["parity"] is not None)
    print(f"{tag} forward parity: worst site {par[1]} rel-L2 {par[0]:.2e}; "
          + " ".join(f"{s['name'].replace('backbone.', '')}={s['parity']:.1e}" for s in shim.sites if s["parity"] is not None))
    sm = max(stats.items(), key=lambda kv: kv[1][0])
    sv = max(stats.items(), key=lambda kv: kv[1][1])
    print(f"{tag} running stats: worst mean {sm[1][0]:.2e} ({sm[0]}), worst var {sv[1][1]:.2e} ({sv[0]}) over {len(stats)} BatchNorms")

    assert shim.inert == (4 if case == "r8_mixed_b64" else 0)  # mask_oracle's pose losses call gdrn_losses on an inert head
    assert len(stats) == 43 and all(nbt for _, _, nbt in stats.values()), stats
    assert not fails, f"{len(fails)} channels above {BOUND[precision]}: {fails[:10]}"
    assert sm[1][0] < STAT_BOUND and sv[1][1] < STAT_BOUND, (sm, sv)
    assert par[0] < PARITY_BOUND, par
