"""The read / rebuild split of the hybrid gradient pass: every split gives exactly the reading pass's result on a shape with a
ragged last column tile, a short last row chunk and a short last row group; and split -1 is chosen from the card's enforced
power limit, with the power-capped value when the limit cannot be read."""

import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import ops

CAPPED, FULL = 2, 5  # the sweeps behind these values are in the comment above kAutoSplitCapped in csrc/evok_grad.cu


@pytest.mark.parametrize("milliwatts, split", [(700_000, FULL), (550_000, FULL), (549_999, CAPPED), (400_000, CAPPED), (0, CAPPED), (-1, CAPPED)])
def test_split_policy_follows_the_power_limit(milliwatts, split):
    assert nat.lib().evok_grad_auto_split(milliwatts) == split


def test_unreadable_power_limit_falls_back_to_the_capped_split():
    lib = nat.lib()
    for device in (-1, 4096):  # no such device: the query reports that it could not read a limit
        assert lib.evok_grad_power_limit_mw(device) == -1
    assert lib.evok_grad_auto_split(-1) == CAPPED
    if not torch.cuda.is_available():
        assert lib.evok_grad_power_limit_mw(0) == -1


# the metric's grid (10 column tiles x 39 row chunks) at a small size: 9800 columns leave 584 in the last 1024-column tile;
# 9001 units make chunks of 231 units, the last one of 223, whose last row group holds 3
SEED, STREAM, ROW0, UNITS, D = 5, 11, 2048, 9001, 9_800


@pytest.mark.gpu
@pytest.mark.parametrize("form_name", ["symmetric", "separable", "exp"])
def test_every_split_is_bit_identical_to_reading_every_row(form_name):
    form = {"symmetric": ops.GRAD_SYMMETRIC, "separable": ops.GRAD_SEPARABLE, "exp": ops.GRAD_EXP}[form_name]
    sym = form == ops.GRAD_SYMMETRIC
    n = 2 * UNITS if sym else UNITS
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(3)
    mu = torch.rand(D, generator=gen, device=dev) * 4.0 - 2.0
    sigma = torch.rand(D, generator=gen, device=dev) * 0.9 + 0.1
    X = torch.empty(n, D, device=dev)
    ops.sample_eval(ops.OBJ_NONE, X, mu, sigma, n_rows=n, symmetric=sym, seed=SEED, stream_id=STREAM, row0=ROW0)
    w = torch.randn(n, generator=gen, device=dev)
    w[7:40] = 0.0  # rows whose weights are both zero are skipped on either path
    ref = ops.grad(form, X, w, mu, sigma, 0.5, 0.25)
    kw = dict(seed=SEED, stream_id=STREAM, row0=ROW0, scale_mu=0.5, scale_sigma=0.25)
    for split in list(range(ops.GRAD_SPLIT_PERIOD + 1)) + [-1]:
        gmu, gsig = ops.grad_hybrid(form, X, w, mu, sigma, split=split, **kw)
        assert torch.equal(gmu, ref[0]) and torch.equal(gsig, ref[1]), split


@pytest.mark.gpu
def test_power_limit_of_the_current_card_maps_to_a_measured_split():
    lib = nat.lib()
    mw = lib.evok_grad_power_limit_mw(torch.cuda.current_device())
    assert mw == -1 or mw > 0
    assert lib.evok_grad_auto_split(mw) in (CAPPED, FULL)
