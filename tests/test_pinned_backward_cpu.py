"""The pinned float64 backward harness (tests/pinned_backward.py) without a GPU.

  * The oracle at B = 2 in float64: pins taken from its own forward, written into the engine's layouts by an encoder independent
    of the harness's decoders (numpy packbits for the NHWC ReLU bitmaps, a scan over the nine window offsets for the max-pool
    codes).  Replayed through the shim, every pin is consumed, no decision differs and the gradients and running statistics
    equal plain autograd's.
  * The decoders against hand-built cases: bit order, max-pool ties, border windows, codes that point into the padding.
  * The comparator flags a planted 1 % error in one row of a 512-row tensor, which a tensor-level rel-L2 would not notice.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import pinned_backward as PB
from gdr_net_b200 import synth
from oracle import fixtures
from oracle import gdrn_oracle as O


# ------------------------------------------------------------------------------------------------ independent encoder
def encode_bitmap(x_nchw: torch.Tensor) -> torch.Tensor:
    """[x > 0] in the engine's layout: flat NHWC element e is bit e & 7 of byte e >> 3."""
    bits = (x_nchw > 0).permute(0, 2, 3, 1).reshape(-1).numpy()
    return torch.from_numpy(np.packbits(bits, bitorder="little"))


def encode_pool(x_nchw: torch.Tensor) -> torch.Tensor:
    """uint8 NHWC window codes dy * 3 + dx of max_pool2d(x, 3, 2, 1): the first strict maximum over dy, then dx."""
    x = x_nchw.numpy()
    B, C, H, W = x.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    pad = np.full((B, C, H + 2, W + 2), -np.inf)
    pad[:, :, 1:-1, 1:-1] = x
    best = np.full((B, C, Ho, Wo), -np.inf)
    code = np.zeros((B, C, Ho, Wo), np.uint8)
    for dy in range(3):
        for dx in range(3):
            v = pad[:, :, dy:dy + 2 * Ho:2, dx:dx + 2 * Wo:2]
            upd = v > best
            best = np.where(upd, v, best)
            code = np.where(upd, dy * 3 + dx, code).astype(np.uint8)
    return torch.from_numpy(np.ascontiguousarray(code.transpose(0, 2, 3, 1)))


class Recorder:
    """torch.nn.functional with the arguments of the decision calls recorded in call order."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return getattr(TF, name)

    def relu(self, x, inplace=False):
        self.calls.append(("relu", x.detach().clone()))
        return TF.relu(x)

    def leaky_relu(self, x, negative_slope=0.01, inplace=False):
        self.calls.append(("leaky_relu", x.detach().clone()))
        return TF.leaky_relu(x, negative_slope)

    def max_pool2d(self, x, *a, **k):
        self.calls.append(("max_pool2d", x.detach().clone()))
        return TF.max_pool2d(x, *a, **k)

    def l1_loss(self, a, b, reduction="mean", **k):
        if a.requires_grad or b.requires_grad:
            self.calls.append(("l1_loss", (a - b).detach().clone()))
        return TF.l1_loss(a, b, reduction=reduction)


def pins_from_oracle(calls):
    """Pins in the engine's layouts from recorded oracle calls: BatchNorm sites as bitmaps, GroupNorm (the three ReLUs after the
    40 BatchNorm ones) and LeakyReLU sites from their outputs, the max-pool as codes, the L1 calls as signs."""
    pins, n_relu = [], 0
    for i, (kind, x) in enumerate(calls):
        name = f"{kind}#{i}"
        if kind == "relu" and n_relu < 40:
            B, C, H, W = x.shape
            pins.append(PB.Pin.relu_bitmap(name, encode_bitmap(x), (B, H, W, C)))
        elif kind == "relu":
            pins.append(PB.Pin.positive("relu", name, TF.relu(x).permute(0, 2, 3, 1)))
        elif kind == "leaky_relu":
            pins.append(PB.Pin.positive("leaky_relu", name, TF.leaky_relu(x, 0.1)))
        elif kind == "max_pool2d":
            B, C, H, W = x.shape
            pins.append(PB.Pin.pool(name, encode_pool(x), (B, H, W, C)))
        else:
            pins.append(PB.Pin.sign(name, torch.sign(x)))
        n_relu += kind == "relu"
    return pins


@pytest.fixture(scope="module")
def oracle_b2():
    sd = fixtures.calibrated_state_dict(0)
    batch = synth.make_batch(2, seed=3)
    fwd = lambda leaf, b: O.gdrn_forward(leaf, b, train=True, do_loss=True, update_stats=True)  # noqa: E731
    rec = Recorder()
    old = O.F
    O.F = rec
    try:
        out, leaf, _ = PB.replay(fwd, sd, batch, None, (O,), device="cpu")
    finally:
        O.F = old
    return sd, batch, fwd, rec.calls, out, leaf


def test_recorded_call_order_is_the_engines(oracle_b2):
    calls = oracle_b2[3]
    kinds = [k for k, _ in calls]
    assert kinds == ["relu", "max_pool2d"] + ["relu"] * 39 + ["relu"] * 3 + ["leaky_relu"] * 2 + ["l1_loss"] * 7
    shapes = [tuple(x.shape) for _, x in calls]
    assert shapes[0] == (2, 64, 128, 128) and shapes[1] == (2, 64, 128, 128) and shapes[40] == (2, 256, 64, 64) and shapes[41] == (2, 128, 32, 32)
    assert shapes[-7:-3] == [(2, 1, 64, 64)] * 3 + [(2, 64, 64)] and shapes[-2:] == [(2, 2), (2,)]
    assert shapes[-3][0] == 2 and shapes[-3][2] == 3  # point matching: [B, n, 3]


def test_pinned_replay_equals_autograd(oracle_b2):
    """Pins from the oracle's own decisions: the pinned float64 step is the plain one, to rounding."""
    sd, batch, fwd, calls, out, leaf = oracle_b2
    pins = pins_from_oracle(calls)
    assert len(pins) == 53
    out_p, leaf_p, shim = PB.replay(fwd, sd, batch, pins, (O,), device="cpu")
    assert len(shim.sites) == 53 and shim.inert == 0
    assert all(s["flips"] == 0 for s in shim.sites), [s for s in shim.sites if s["flips"]]
    for k, v in out["losses"].items():
        assert abs(float(out_p["losses"][k].detach()) - float(v.detach())) <= 1e-12 * abs(float(v)), k
    worst, worst_rel = 0.0, 0.0
    for name, t in leaf.items():
        if isinstance(t, torch.Tensor) and t.requires_grad:
            e, rel = PB.row_errors(leaf_p[name].grad, t.grad)
            worst, worst_rel = max(worst, float(e.max())), max(worst_rel, rel)
        elif name.endswith(("running_mean", "running_var")):
            assert float((leaf_p[name] - t).abs().max()) <= 1e-12 * float(t.abs().max()), name
        elif name.endswith("num_batches_tracked"):
            assert int(leaf_p[name]) == int(t) == int(sd[name]) + 1, name
    # measured: rel-L2 <= 4e-13 per tensor; rows whose gradient is a cancelling sum (BatchNorm, GroupNorm entries) reach 5e-10
    print(f"pinned vs plain autograd, float64 B = 2: worst rel-L2 {worst_rel:.1e}, worst per-row error {worst:.1e}")
    assert worst_rel < 2e-12 and worst < 1e-8


def test_every_pin_must_be_consumed_and_match(oracle_b2):
    sd, batch, fwd, calls, _, _ = oracle_b2
    pins = pins_from_oracle(calls)
    with pytest.raises(AssertionError, match="not consumed"):
        PB.replay(fwd, sd, batch, pins + [PB.Pin.sign("extra", torch.zeros(2))], (O,), device="cpu")
    bad = list(pins)
    bad[3] = PB.Pin.relu_bitmap("wrong", torch.zeros(2 * 64 * 64 * 64 // 8, dtype=torch.uint8), (2, 64, 64, 32))
    with pytest.raises(AssertionError, match="shape"):
        PB.replay(fwd, sd, batch, bad, (O,), device="cpu")


def test_flipped_decisions_are_counted(oracle_b2):
    """A pin that disagrees with the float64 forward is followed, and counted."""
    sd, batch, fwd, calls, _, _ = oracle_b2
    pins = pins_from_oracle(calls)
    B, C, H, W = calls[2][1].shape
    inv = encode_bitmap(calls[2][1]) ^ 0x01  # element 0 of every byte flipped
    pins[2] = PB.Pin.relu_bitmap("flipped", inv, (B, H, W, C))
    _, _, shim = PB.replay(fwd, sd, batch, pins, (O,), device="cpu", parity=False)
    assert shim.sites[2]["flips"] == B * C * H * W // 8


# ------------------------------------------------------------------------------------------------ decoders, hand-built
def test_bitmap_bit_order():
    # NHWC [1, 2, 2, 4]: flat e = ((h * 2) + w) * 4 + c; set e = 2, 9 and 15
    bits = torch.tensor([0b00000100, 0b10000010], dtype=torch.uint8)
    m = PB.unpack_bitmap(bits, (1, 2, 2, 4))
    assert m.shape == (1, 4, 2, 2)
    on = {tuple(i) for i in m.nonzero().tolist()}
    # e = 2 -> h 0 w 0 c 2;  e = 9 -> h 1 w 0 c 1;  e = 15 -> h 1 w 1 c 3
    assert on == {(0, 2, 0, 0), (0, 1, 1, 0), (0, 3, 1, 1)}
    x = torch.randn(2, 16, 5, 8, dtype=torch.float64)
    assert torch.equal(PB.unpack_bitmap(encode_bitmap(x), (2, 5, 8, 16)), x > 0)


def test_pool_codes_ties_and_borders():
    x = torch.tensor([[[[1.0, 5.0, 5.0, 0.0],
                        [5.0, 2.0, 0.0, 0.0],
                        [3.0, 3.0, 3.0, 3.0],
                        [0.0, 0.0, 7.0, 7.0]]]], dtype=torch.float64)
    # windows start at (2 oy - 1, 2 ox - 1); row dy = 0 / column dx = 0 of the top / left windows are padding
    # (0,0): rows -1..1, cols -1..1: max 5 at (0,1) and (1,0) -> first is (0,1): dy 1 dx 2 -> 5
    # (0,1): rows -1..1, cols 1..3: 5 at (0,1) and (0,2) -> (0,1): dy 1 dx 0 -> 3
    # (1,0): rows 1..3, cols -1..1: 5 at (1,0): dy 0 dx 1 -> 1
    # (1,1): rows 1..3, cols 1..3: 7 at (3,2) and (3,3) -> (3,2): dy 2 dx 1 -> 7
    want = torch.tensor([[[[5, 3], [1, 7]]]])
    arg = encode_pool(x)
    assert torch.equal(arg.permute(0, 3, 1, 2).long(), want)
    assert torch.equal(PB.first_max_codes(x), want)
    xg = x.clone().requires_grad_(True)
    y = PB.pool_gather(xg, PB.pool_codes(arg))
    assert torch.equal(y.detach(), TF.max_pool2d(x, 3, 2, 1))
    y.sum().backward()
    g = torch.zeros_like(x)
    g[0, 0, 0, 1] = 2.0  # chosen by two windows
    g[0, 0, 1, 0] = 1.0
    g[0, 0, 3, 2] = 1.0
    assert torch.equal(xg.grad, g)
    with pytest.raises(AssertionError, match="padding"):
        PB.pool_gather(x, torch.tensor([[[[0, 3], [1, 7]]]]))  # code 0 of window (0,0) is the padded corner


def test_pool_codes_random_against_torch():
    x = torch.randn(2, 8, 9, 12, dtype=torch.float64)
    x[0, 0, :4, :4] = 0.0  # ties
    codes = PB.pool_codes(encode_pool(x))
    assert torch.equal(codes, PB.first_max_codes(x))
    assert torch.equal(PB.pool_gather(x, codes), TF.max_pool2d(x, 3, 2, 1))


# ------------------------------------------------------------------------------------------------ comparator
def test_comparator_flags_one_row_at_one_percent():
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(512, 256, 3, 3, generator=g, dtype=torch.float64)
    noisy = ref + 1e-4 * ref.flatten(1).norm(dim=1).view(-1, 1, 1, 1) / 48 * torch.randn(ref.shape, generator=g, dtype=torch.float64)
    fails, table = PB.compare_grads({"w": noisy}, {"w": ref}, 5e-3)
    assert not fails and table[0][2] < 2e-4
    bad = noisy.clone()
    d = torch.randn(256, 3, 3, generator=g, dtype=torch.float64)
    bad[137] += 0.01 * ref[137].norm() * d / d.norm()
    fails, table = PB.compare_grads({"w": bad}, {"w": ref}, 5e-3)
    assert [f[:2] for f in fails] == [("w", 137)] and 0.009 < fails[0][2] < 0.011
    assert table[0][3] < 1e-3  # the tensor-level rel-L2 of the same error: 0.01 / sqrt(512)
    nan = noisy.clone()
    nan[3, 0, 0, 0] = float("nan")
    assert [f[:2] for f in PB.compare_grads({"w": nan}, {"w": ref}, 5e-3)[0]] == [("w", 3)]


def test_comparator_floor_and_one_d():
    ref = torch.tensor([1.0, 1e-9, -2.0, 0.0], dtype=torch.float64)
    got = ref + torch.tensor([0.0, 1e-9, 0.0, 1e-7], dtype=torch.float64)
    e, rel = PB.row_errors(got, ref)
    floor = 1e-3 * float(ref.norm()) / 2
    assert torch.allclose(e, torch.tensor([0.0, 1e-9 / floor, 0.0, 1e-7 / floor], dtype=torch.float64))
    # with a 1-D bound the entries are measured against 0.1 of the RMS entry: a 2 % error of a typical entry is flagged, the
    # same absolute error on an entry that is 1e-3 of the RMS one is not
    g = torch.Generator().manual_seed(1)
    ref = torch.randn(128, generator=g, dtype=torch.float64)
    ref[7] = 1e-3 * ref.norm() / 128 ** 0.5
    got = ref.clone()
    got[7] += 0.002 * ref.norm() / 128 ** 0.5  # e_r 0.02 against 0.1 of the RMS entry
    assert not PB.compare_grads({"b": got}, {"b": ref}, 1e-3, 0.05)[0]
    assert PB.compare_grads({"b": got}, {"b": ref}, 1e-3)[0]  # against the row floor it would be
    ref[3] = ref.norm() / 128 ** 0.5
    got = ref.clone()
    got[3] *= 1.02
    assert [f[:2] for f in PB.compare_grads({"b": got}, {"b": ref}, 1e-3, 1e-2)[0]] == [("b", 3)]


def test_family_names():
    assert PB.family("backbone.conv1.weight") == "backbone.stem/conv.weight"
    assert PB.family("backbone.bn1.bias") == "backbone.stem/bn.bias"
    assert PB.family("backbone.layer3.1.bn2.weight") == "backbone.layer3/bn.weight"
    assert PB.family("backbone.layer2.0.downsample.1.weight") == "backbone.layer2/bn.weight"
    assert PB.family("backbone.layer2.0.downsample.0.weight") == "backbone.layer2/conv.weight"
    assert PB.family("rot_head_net.features.21.weight") == "rot_head_net/bn.weight"
    assert PB.family("rot_head_net.features.23.bias") == "rot_head_net/conv.bias"
    assert PB.family("pnp_net.features.4.bias") == "pnp_net/gn.bias"
    assert PB.family("pnp_net.fc_r.weight") == "pnp_net/fc.weight"
