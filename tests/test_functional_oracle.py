"""The float64 statement of the functional tells (oracle/functional_oracle.py) checked on the CPU, two ways: against the real
reference's outputs (tests/golden/functional_golden.npz, including the CEM edges where the reference gives NaN) and against this
package's own generic torch path of the same functions run in float64 (on the CPU the functional API takes that path).
tests/test_functional_batched.py then holds the CUDA kernels to this oracle."""

import os
import zlib

import numpy as np
import pytest
import torch

from evotorch_b200.algorithms import functional as F
from oracle import functional_oracle as FO

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "functional_golden.npz"))
RANKINGS = ["centered", "linear", "nes", "normalized", "raw"]


def _close(got, want, rtol, atol=0.0):
    np.testing.assert_allclose(np.asarray(got, np.float64), np.asarray(want, np.float64), rtol=rtol, atol=atol, equal_nan=True)


# ------------------------------------------------------------------------------------------------ against the reference
OPT_CFG = {
    "clipup": (dict(lr=[0.15], momentum=[0.9], max_speed=[0.3]), dict(lr=[0.1, 0.2, 0.3], momentum=[0.9] * 3, max_speed=[0.15, 0.5, 0.45])),
    "adam": (dict(lr=[0.05], beta1=[0.9]), dict(lr=[0.01, 0.05, 0.1], beta1=[0.8] * 3)),
    "sgd": (dict(lr=[0.1], momentum=[0.5]), dict(lr=[0.1, 0.2, 0.3], momentum=[0.0] * 3)),
}


@pytest.mark.parametrize("name", list(OPT_CFG))
@pytest.mark.parametrize("tag", ["plain", "batched"])
def test_oracle_optimizer_tells_match_reference(name, tag):
    """Five tells of each functional optimizer, per item with per-item hyper-parameters."""
    cfg = OPT_CFG[name][tag == "batched"]
    c0 = GOLD["opt/c0"] if tag == "plain" else GOLD["opt/c0_b"]
    grads = GOLD["opt/grads"] if tag == "plain" else GOLD["opt/grads_b"]
    c0 = np.atleast_2d(c0).astype(np.float64)
    for b in range(c0.shape[0]):
        center, vel, m, v, t = c0[b], np.zeros_like(c0[b]), np.zeros_like(c0[b]), np.zeros_like(c0[b]), 0
        for g, want in zip(grads, GOLD[f"opt/{name}/{tag}/centers"]):
            gb = np.atleast_2d(g)[b]
            if name == "clipup":
                r = FO.clipup_tell(center, vel, gb, lr=cfg["lr"][b], momentum=cfg["momentum"][b], max_speed=cfg["max_speed"][b])
                vel = r["velocity"]
            elif name == "adam":
                r = FO.adam_tell(center, m, v, t, gb, lr=cfg["lr"][b], beta1=cfg["beta1"][b])
                m, v, t = r["m"], r["v"], r["t"]
            else:
                r = FO.sgd_tell(center, vel, gb, lr=cfg["lr"][b], momentum=cfg["momentum"][b])
                vel = r["velocity"]
            center = r["center"]
            _close(center, np.atleast_2d(want)[b], rtol=2e-6, atol=2e-6)


PGPE_GOLD = {
    # tag: (optimizer, optimizer kwargs per item, stdev lr, ranking, maximize, symmetric, stdev_min, stdev_max, stdev_max_change)
    "sym_clipup": ("clipup", [dict(lr=0.3, momentum=0.9, max_speed=0.6)], 0.1, "centered", False, True, 0.0, np.inf, 0.2),
    "nonsym_adam_nes": ("adam", [dict(lr=0.05)], 0.1, "nes", False, False, 0.0, np.inf, np.inf),
    "sym_sgd_linear_max": ("sgd", [dict(lr=0.1)], 0.2, "linear", True, True, 0.5, 1.0, 0.1),
    "batched": ("clipup", [dict(lr=0.2, momentum=0.9, max_speed=0.4), dict(lr=0.4, momentum=0.9, max_speed=0.8)], 0.1, "centered", False, True,
                0.0, np.inf, 0.2),
}


def _opt_step(name, center, state, g, kw):
    if name == "clipup":
        r = FO.clipup_tell(center, state.get("v", np.zeros_like(center)), g, **kw)
        return r["center"], {"v": r["velocity"]}
    if name == "adam":
        r = FO.adam_tell(center, state.get("m", np.zeros_like(center)), state.get("vv", np.zeros_like(center)), state.get("t", 0), g, **kw)
        return r["center"], {"m": r["m"], "vv": r["v"], "t": r["t"]}
    r = FO.sgd_tell(center, state.get("v", np.zeros_like(center)), g, **kw)
    return r["center"], {"v": r["velocity"]}


@pytest.mark.parametrize("tag", list(PGPE_GOLD))
def test_oracle_pgpe_tells_match_reference(tag):
    """Four generations of the reference's functional PGPE replayed through the oracle from the populations it drew."""
    opt, opt_kw, lr_sigma, method, maximize, sym, lo, hi, mc = PGPE_GOLD[tag]
    centers = np.atleast_2d(GOLD[f"pgpe/{tag}/center0"]).astype(np.float64)
    stdevs = np.broadcast_to(GOLD[f"pgpe/{tag}/stdev0"], centers.shape).astype(np.float64)
    states = [{} for _ in range(centers.shape[0])]
    for g in range(GOLD[f"pgpe/{tag}/values"].shape[0]):
        values = GOLD[f"pgpe/{tag}/values"][g].reshape((centers.shape[0],) + GOLD[f"pgpe/{tag}/values"].shape[-2:])
        evals = GOLD[f"pgpe/{tag}/evals"][g].reshape(centers.shape[0], -1)
        for b in range(centers.shape[0]):
            gr = FO.pgpe_gradients(values[b], evals[b], centers[b], stdevs[b], ranking_method=method, maximize=maximize, symmetric=sym)
            stdevs[b], _ = FO.sigma_update(stdevs[b], gr["sigma"], lr_sigma, stdev_min=np.full(centers.shape[1], lo, np.float32),
                                           stdev_max=np.full(centers.shape[1], hi, np.float32),
                                           stdev_max_change=np.full(centers.shape[1], mc, np.float32))
            centers[b], states[b] = _opt_step(opt, centers[b], states[b], gr["mu"], opt_kw[b])
        _close(centers, np.atleast_2d(GOLD[f"pgpe/{tag}/center"][g]), rtol=1e-5, atol=1e-5)
        _close(stdevs, np.atleast_2d(GOLD[f"pgpe/{tag}/stdev"][g]), rtol=1e-5, atol=1e-5)


CEM_GOLD = {
    # tag: (parenthood ratio, maximize, stdev_min, stdev_max, stdev_max_change)
    "plain": (0.25, False, 0.0, np.inf, 0.3),
    "max_bounds": (0.5, True, 0.4, 1.5, np.inf),
    "batched": (0.25, False, 0.0, np.inf, np.inf),
    "one_elite": (0.03, False, 0.0, np.inf, np.inf),
    "zero_elites": (0.01, True, 0.0, np.inf, np.inf),
    "zero_stdev": (0.25, False, 0.0, np.inf, np.inf),
}


@pytest.mark.parametrize("tag", list(CEM_GOLD))
def test_oracle_cem_tells_match_reference(tag):
    """The reference's functional CEM replayed through the oracle, the NaN edges included: one elite (std of one row), no elite, and a
    zero stdev with an unlimited max change (|0| * inf = NaN through torch.max / torch.min)."""
    ratio, maximize, lo, hi, mc = CEM_GOLD[tag]
    centers = np.atleast_2d(GOLD[f"cem/{tag}/center0"]).astype(np.float64)
    stdevs = np.broadcast_to(GOLD[f"cem/{tag}/stdev0"], centers.shape).astype(np.float64).copy()
    D = centers.shape[1]
    bounds = dict(stdev_min=np.full(D, lo, np.float32), stdev_max=np.full(D, hi, np.float32), stdev_max_change=np.full(D, mc, np.float32))
    for g in range(GOLD[f"cem/{tag}/values"].shape[0]):
        values = GOLD[f"cem/{tag}/values"][g].reshape((centers.shape[0],) + GOLD[f"cem/{tag}/values"].shape[-2:])
        evals = GOLD[f"cem/{tag}/evals"][g].reshape(centers.shape[0], -1)
        for b in range(centers.shape[0]):
            r = FO.cem_tell(values[b], evals[b], centers[b], stdevs[b], parenthood_ratio=ratio, maximize=maximize, **bounds)
            centers[b], stdevs[b] = r["center"], r["stdev"]
        _close(centers, np.atleast_2d(GOLD[f"cem/{tag}/center"][g]), rtol=1e-5, atol=1e-5)
        _close(stdevs, np.atleast_2d(GOLD[f"cem/{tag}/stdev"][g]), rtol=1e-5, atol=2e-5)
    if tag in ("one_elite", "zero_elites"):
        assert np.isnan(stdevs).all()
    if tag == "zero_stdev":
        assert np.isnan(stdevs[:, 1::2]).all() and np.isfinite(stdevs[:, 0::2]).all()


# ------------------------------------------------------------------------------------------------ against the float64 torch path
def _T(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64)


def _opt_config(opt, lrs):
    """optimizer_config of `pgpe` besides the (per-item) learning rate"""
    if opt == "clipup":
        return dict(momentum=0.8, max_speed=_T(np.asarray(lrs) * 1.5))
    if opt == "adam":
        return dict(beta1=0.85)
    return dict(momentum=0.6)


@pytest.mark.parametrize("opt", ["clipup", "adam", "sgd"])
@pytest.mark.parametrize("ranking", RANKINGS)
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("sense", ["min", "max"])
def test_oracle_pgpe_tell_matches_the_float64_torch_path(opt, ranking, symmetric, sense):
    """Three tells of three batch items with per-item learning rates, a batched stdev, bounds and a max change: the oracle, fed the
    same float64 inputs, agrees with F.pgpe_tell on the CPU in float64.  The oracle ranks in fp32 (as the reference and the kernels
    do), the torch path in float64, hence the 1e-6 relative bound on the utilities' scale."""
    rng = np.random.default_rng(zlib.crc32(f"{opt}/{ranking}/{symmetric}/{sense}".encode()))
    B, N, D = 3, 16, 5
    lrs = [0.05, 0.1, 0.2]
    center0 = rng.uniform(-2, 2, (B, D))
    stdev0 = rng.uniform(0.5, 1.5, (B, D))
    state = F.pgpe(center_init=_T(center0), center_learning_rate=_T(lrs), stdev_learning_rate=0.2, objective_sense=sense,
                   ranking_method=ranking, optimizer=opt, optimizer_config=_opt_config(opt, lrs),
                   stdev_init=_T(stdev0), stdev_min=0.6, stdev_max=1.4, stdev_max_change=0.15, symmetric=symmetric)
    centers, stdevs = center0.copy(), stdev0.copy()
    ostates = [{} for _ in range(B)]
    for _ in range(3):
        Z = rng.standard_normal((B, N // 2 if symmetric else N, D))
        X = np.empty((B, N, D))
        if symmetric:
            X[:, 0::2], X[:, 1::2] = centers[:, None] + stdevs[:, None] * Z, centers[:, None] - stdevs[:, None] * Z
        else:
            X = centers[:, None] + stdevs[:, None] * Z
        X = X.astype(np.float32).astype(np.float64)  # the oracle ranks fp32 data: keep the inputs exactly representable
        f = np.round((X**2).sum(-1) * 8) / 8  # with ties
        state = F.pgpe_tell(state, _T(X), _T(f))
        for b in range(B):
            gr = FO.pgpe_gradients(X[b], f[b], centers[b], stdevs[b], ranking_method=ranking, maximize=(sense == "max"), symmetric=symmetric)
            stdevs[b], _ = FO.sigma_update(stdevs[b], gr["sigma"], 0.2, stdev_min=0.6, stdev_max=1.4, stdev_max_change=0.15)
            kw = {"clipup": dict(lr=lrs[b], momentum=0.8, max_speed=1.5 * lrs[b]), "adam": dict(lr=lrs[b], beta1=0.85),
                  "sgd": dict(lr=lrs[b], momentum=0.6)}[opt]
            centers[b], ostates[b] = _opt_step(opt, centers[b], ostates[b], gr["mu"], kw)
        _close(state.optimizer_state.center.numpy(), centers, rtol=1e-5, atol=1e-6)
        _close(state.stdev.numpy(), stdevs, rtol=1e-5, atol=1e-6)
        # and take the torch path's state as the next starting point, so that errors do not compound over the tells
        centers, stdevs = state.optimizer_state.center.numpy().copy(), state.stdev.numpy().copy()


@pytest.mark.parametrize("ratio", [0.0625, 0.125, 0.5, 1.0])
@pytest.mark.parametrize("sense", ["min", "max"])
def test_oracle_cem_tell_matches_the_float64_torch_path(ratio, sense):
    """F.cem_tell in float64 on the CPU against the oracle's two-pass elite moments (E = 1, 2, 8, 16 of N = 16), batched, with bounds.
    E = 1 gives a NaN stdev on both sides."""
    rng = np.random.default_rng(int(ratio * 1000) + (sense == "max"))
    B, N, D = 4, 16, 6
    center0 = rng.uniform(-2, 2, (B, D))
    stdev0 = rng.uniform(0.5, 1.5, (B, D))
    X = (center0[:, None] + stdev0[:, None] * rng.standard_normal((B, N, D))).astype(np.float32).astype(np.float64)
    f = np.round((X**2).sum(-1) * 4) / 4
    st = F.cem(center_init=_T(center0), parenthood_ratio=ratio, objective_sense=sense, stdev_init=_T(stdev0), stdev_min=0.3, stdev_max=2.0,
               stdev_max_change=0.5)
    new = F.cem_tell(st, _T(X), _T(f))
    for b in range(B):
        r = FO.cem_tell(X[b], f[b], center0[b], stdev0[b], parenthood_ratio=ratio, maximize=(sense == "max"), stdev_min=0.3, stdev_max=2.0,
                        stdev_max_change=0.5)
        _close(new.center[b].numpy(), r["center"], rtol=1e-12, atol=1e-12)
        _close(new.stdev[b].numpy(), r["stdev"], rtol=1e-6, atol=1e-7)
        assert np.isnan(r["stdev"]).all() == (r["num_elites"] == 1)


def test_oracle_zero_stdev_with_unlimited_change_is_nan_as_in_torch():
    """modify_tensor with a zero original and an infinite max change: |0| * inf = NaN, kept by torch.max / torch.min, in the torch
    path and in the oracle; a finite max change keeps the zero."""
    from evotorch_b200.tools import modify_tensor

    s = np.array([0.0, 1.0])
    got = modify_tensor(_T(s), _T([0.5, 1.2]), lb=_T([0.0, 0.0]), ub=_T([np.inf, np.inf]), max_change=_T([np.inf, np.inf])).numpy()
    want, _ = FO.sigma_update(s, np.array([0.5, 0.2]), 1.0, stdev_min=0.0, stdev_max=np.inf, stdev_max_change=np.inf)
    _close(got, [np.nan, 1.2], rtol=1e-7)
    _close(want, [np.nan, 1.2], rtol=1e-7)
    kept, _ = FO.sigma_update(s, np.array([0.5, 0.2]), 1.0, stdev_max_change=0.2)
    _close(kept, [0.0, 1.2], rtol=1e-7)
