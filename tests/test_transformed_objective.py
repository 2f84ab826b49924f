"""Objectives of the transformed row y = M (x - o) on the CPU: the parsing and validation of the `transform` keyword and of y / yn,
the torch function against the float64 oracle (oracle/transformed_objective_oracle.py) with shared and per-item transforms, pickling
and with_data, the sources of the same expressions without a transform (pinned by a golden), and the C ABI's return codes."""

import ctypes
import json
import math
import os
import pickle

import numpy as np
import pytest
import torch

from evotorch_b200 import _native as nat
from evotorch_b200 import jit
from evotorch_b200.objectives import FusedObjective
from oracle import transformed_objective_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transformed_twin_objective_sources.json")

ELLIPSOID = "10**(6 * j / maximum(D - 1, 1)) * y**2"
# name -> (FusedObjective keywords without the transform, oracle function, data maker (B, D) or None)
SPECS = {
    "rot_ellipsoid": (dict(sums={"s": ELLIPSOID}, value="s"), O.rot_ellipsoid, None),
    "rot_rastrigin": (dict(sums={"s": "y**2 - 10 * cos(2 * pi * y)"}, value="10 * D + s"), O.rot_rastrigin, None),
    "rot_rosenbrock": (dict(sums={"s": "100 * (yn - y**2)**2 + (1 - y)**2"}, value="s"), O.rot_rosenbrock, None),
    "rot_schwefel_1_2": (dict(running={"c": "y"}, sums={"s": "c**2"}, value="s"), O.rot_schwefel_1_2, None),
    "lunacek_like": (dict(sums={"a": "(2 * sg * x - 2.5)**2", "b": "(2 * sg * x - mu1)**2", "c": "cos(2 * pi * y)",
                                "p": "maximum(0, abs(x) - 5)**2"},
                          value="minimum(a, D + s * b) + 10 * (D - c) + 1e4 * p"), O.lunacek_like, "lunacek"),
    "penalised_ellipsoid": (dict(sums={"s": ELLIPSOID, "p": "maximum(0, abs(x) - 5)**2"}, value="s + 100 * p"), O.penalised_ellipsoid, None),
}


def lunacek_data(batch: tuple, D: int, gen: torch.Generator, device="cpu") -> dict:
    sg = torch.where(torch.rand(batch + (D,), generator=gen) < 0.5, -1.0, 1.0)
    s = torch.full(batch + (1,), 1 - 1 / (2 * math.sqrt(D + 20) - 8.2))
    mu1 = -torch.sqrt((2.5**2 - 1) / s)
    return {"sg": sg.to(device), "mu1": mu1.to(device), "s": s.to(device)}


def make(name: str, M: torch.Tensor, o: torch.Tensor, gen: torch.Generator, **extra) -> tuple:
    """(objective, the oracle's function of X) of SPECS[name] on the transform (M, o)."""
    kw, fn, data = SPECS[name]
    batch, D = tuple(M.shape[:-2]), M.shape[-1]
    if data:
        d = lunacek_data(batch, D, gen, M.device)
        obj = FusedObjective(name, data=d, transform=(M, o), **kw, **extra)
        return obj, lambda X: fn(X, M.cpu(), o.cpu(), d["sg"].cpu(), d["mu1"].cpu(), d["s"].cpu())
    return FusedObjective(name, transform=(M, o), **kw, **extra), lambda X: fn(X, M.cpu(), o.cpu())


def twin_keywords(name: str) -> dict:
    """SPECS[name] with x in place of y and xn in place of yn: the same objective without its transform."""
    kw = SPECS[name][0]
    sub = lambda t: t.replace("yn", "xn").replace("y", "x")  # noqa: E731
    return {k: ({n: sub(t) for n, t in v.items()} if isinstance(v, dict) else sub(v)) for k, v in kw.items()}


def transform(batch: tuple, D: int, gen: torch.Generator, kind: str = "rotation") -> tuple:
    if kind == "rotation":
        M = torch.linalg.qr(torch.randn(batch + (D, D), generator=gen, dtype=torch.float64))[0].float()
    else:  # a general matrix: a rotation times a diagonal scaling times a rotation
        Q = torch.linalg.qr(torch.randn(batch + (D, D), generator=gen, dtype=torch.float64))[0]
        L = torch.diag_embed(10 ** torch.linspace(0, 1, D, dtype=torch.float64).expand(batch + (D,)))
        M = (Q @ L @ Q.mT).float()
    o = 8 * torch.rand(batch + (D,), generator=gen) - 4
    return M, o


# ------------------------------------------------------------------------------------------------ the torch function
@pytest.mark.parametrize("name", list(SPECS))
@pytest.mark.parametrize("D", [1, 2, 3, 33])
@pytest.mark.parametrize("per_item", [False, True])
def test_torch_fn_against_oracle(name, D, per_item):
    gen = torch.Generator().manual_seed(D * 101 + per_item)
    B, n = 3, 5
    M, o = transform((B,) if per_item else (), D, gen, "general" if name == "rot_rastrigin" else "rotation")
    obj, ref = make(name, M, o, gen)
    X = (torch.rand(B, n, D, generator=gen, dtype=torch.float64) * 12 - 6)
    got = obj(X)
    assert got.dtype == torch.float64 and tuple(got.shape) == (B, n)
    np.testing.assert_allclose(got.numpy(), ref(X.numpy()), rtol=1e-12, atol=1e-9)
    assert obj.evok_objective_id is None  # no fused sampler, ever


def test_transform_of_M_alone_has_zero_offset():
    gen = torch.Generator().manual_seed(1)
    M, _ = transform((), 4, gen)
    obj = FusedObjective("e", sums={"s": "y**2"}, value="s", transform=M)
    X = torch.randn(6, 4, generator=gen, dtype=torch.float64)
    np.testing.assert_allclose(obj(X).numpy(), (O.transformed(X.numpy(), M, np.zeros(4)) ** 2).sum(-1), rtol=1e-12)


def test_row_at_offset_is_value_at_zero():
    gen = torch.Generator().manual_seed(2)
    M, o = transform((), 10, gen, "general")
    obj, _ = make("rot_ellipsoid", M * 1e3, o, gen)
    assert obj(o.double()[None])[0].item() == 0.0


# ------------------------------------------------------------------------------------------------ validation
def test_y_without_transform_raises():
    with pytest.raises(ValueError, match="unknown name 'y'"):
        FusedObjective("t", sums={"s": "y**2"}, value="s")
    with pytest.raises(ValueError, match="unknown name 'yn'"):
        FusedObjective("t", sums={"s": "(yn - x)**2"}, value="s")


def test_transform_no_term_reads_raises():
    with pytest.raises(ValueError, match="no term reads y"):
        FusedObjective("t", sums={"s": "x**2"}, value="s", transform=torch.eye(3))


@pytest.mark.parametrize("M, o, what", [
    (torch.zeros(3, 4), None, "square"),
    (torch.zeros(3, 3, dtype=torch.float64), None, "square float32"),
    (torch.eye(3), torch.zeros(4), "o must be"),
    (torch.eye(3), torch.zeros(3, dtype=torch.float64), "o must be"),
])
def test_bad_transform_shapes_raise(M, o, what):
    with pytest.raises(ValueError, match=what):
        FusedObjective("t", sums={"s": "y**2"}, value="s", transform=M if o is None else (M, o))


def test_batch_shapes_must_agree():
    with pytest.raises(ValueError, match="one batch shape"):
        FusedObjective("t", sums={"s": "y**2"}, value="s", transform=(torch.eye(3).expand(2, 3, 3), torch.zeros(5, 3)))
    with pytest.raises(ValueError, match="one batch shape"):
        FusedObjective("t", sums={"s": "w * y**2"}, value="s", data={"w": torch.ones(4, 3)}, transform=torch.eye(3).expand(2, 3, 3))
    ok = FusedObjective("t", sums={"s": "w * y**2"}, value="s", data={"w": torch.ones(2, 3)}, transform=(torch.eye(3).expand(2, 3, 3), torch.zeros(3)))
    assert tuple(ok.data_batch_shape) == (2,)


def test_devices_must_agree():
    meta = torch.eye(3, device="meta")
    with pytest.raises(ValueError, match="o on"):
        FusedObjective("t", sums={"s": "y**2"}, value="s", transform=(meta, torch.zeros(3)))
    with pytest.raises(ValueError, match="different devices"):
        FusedObjective("t", sums={"s": "w * y**2"}, value="s", data={"w": torch.ones(3)}, transform=meta)


def test_y_names_are_reserved_with_a_transform():
    with pytest.raises(ValueError, match="transformed row"):
        FusedObjective("t", sums={"y": "y**2"}, value="y", transform=torch.eye(3))
    with pytest.raises(ValueError, match="transformed row"):
        FusedObjective("t", sums={"s": "y**2 + yn"}, value="s", data={"yn": torch.ones(1)}, transform=torch.eye(3))


def test_pair_terms_and_noise():
    obj = FusedObjective("t", sums={"s": "(yn - y)**2", "q": "y**2 + x"}, value="s + q", transform=torch.eye(3))
    assert obj._spec.pairs == frozenset({"s"})
    with pytest.raises(ValueError, match="rand"):
        FusedObjective("t", sums={"s": "(yn - y)**2 + randn()"}, value="s", transform=torch.eye(3))
    with pytest.raises(ValueError, match="unknown name 'yn'"):
        FusedObjective("t", running={"c": "yn"}, sums={"s": "c**2 + y"}, value="s", transform=torch.eye(3))


# ------------------------------------------------------------------------------------------------ binding, pickling
def test_pickle_round_trip_and_repr():
    gen = torch.Generator().manual_seed(3)
    M, o = transform((2,), 5, gen)
    obj, ref = make("lunacek_like", M, o, gen)
    twin = pickle.loads(pickle.dumps(obj))
    X = torch.randn(2, 4, 5, generator=gen, dtype=torch.float64)
    np.testing.assert_array_equal(twin(X).numpy(), obj(X).numpy())
    assert torch.equal(twin.transform[0], M) and torch.equal(twin.transform[1], o)
    assert "transform=(M (2, 5, 5), o (2, 5))" in repr(obj)
    plain = FusedObjective("r", running={"c": "y"}, sums={"s": "c**2"}, value="s", transform=(M[0], o[0]))
    np.testing.assert_array_equal(pickle.loads(pickle.dumps(plain))(X).numpy(), plain(X).numpy())


def test_with_data_keeps_or_swaps_the_transform():
    gen = torch.Generator().manual_seed(4)
    M, o = transform((), 4, gen)
    M2, o2 = transform((), 4, gen)
    obj = FusedObjective("w", sums={"s": "w * y**2"}, value="s", data={"w": torch.ones(4)}, transform=(M, o))
    X = torch.randn(7, 4, generator=gen, dtype=torch.float64)
    w2 = torch.full((4,), 2.0)
    kept = obj.with_data(w=w2)
    np.testing.assert_allclose(kept(X).numpy(), 2 * obj(X).numpy(), rtol=1e-12)
    swapped = obj.with_data(w=w2, transform=(M2, o2))
    np.testing.assert_allclose(swapped(X).numpy(), 2 * (O.transformed(X.numpy(), M2, o2) ** 2).sum(-1), rtol=1e-12)
    assert kept.source == obj.source == swapped.source
    nodata = FusedObjective("n", sums={"s": "y**2"}, value="s", transform=(M, o))
    np.testing.assert_allclose(nodata.with_data(transform=(M2, o2))(X).numpy(), (O.transformed(X.numpy(), M2, o2) ** 2).sum(-1), rtol=1e-12)
    untransformed = FusedObjective("u", sums={"s": "x**2"}, value="s")
    with pytest.raises(ValueError, match="no transform"):
        untransformed.with_data(transform=M)


def test_in_place_update_reaches_torch_fn():
    gen = torch.Generator().manual_seed(5)
    M, o = transform((), 3, gen)
    obj = FusedObjective("u", sums={"s": "y**2"}, value="s", transform=(M.clone(), o.clone()))
    X = torch.randn(4, 3, generator=gen, dtype=torch.float64)
    obj.transform[1].copy_(o + 1)
    np.testing.assert_allclose(obj(X).numpy(), (O.transformed(X.numpy(), M, o + 1) ** 2).sum(-1), rtol=1e-12)


# ------------------------------------------------------------------------------------------------ sources
def test_transformed_source_declares_the_transform():
    obj = FusedObjective("t", sums={"s": "(yn - y)**2"}, value="s", transform=torch.eye(3))
    assert "static constexpr bool kTransform = true;" in obj.source
    assert "void add_pair(float x, float xn, float y, float yn, int64_t j)" in obj.source


def test_untransformed_twin_sources_are_unchanged():
    """The same expressions without the transform (x for y): their sources, which key the compile cache, are those of the
    language without transforms, pinned in a golden written before transforms existed."""
    with open(GOLDEN) as fh:
        golden = json.load(fh)
    assert set(golden) == set(SPECS)
    for name in SPECS:
        kw = twin_keywords(name)
        kinds = jit.data_kinds(lunacek_data((), 5, torch.Generator().manual_seed(0))) if SPECS[name][2] else None
        spec = jit.ObjectiveSpec(kw.pop("sums", None), kw.pop("value"), kinds, **kw)
        assert spec.source == golden[name], name
        assert "kTransform" not in spec.source


# ------------------------------------------------------------------------------------------------ C ABI, no launch
def _register_transform_id() -> int:
    obj = FusedObjective("abi", sums={"s": "y**2"}, value="s", transform=torch.eye(3))
    return jit._transform_cache[obj.source].objective_id


def test_abi_return_codes():
    lib = nat.lib()
    tid = _register_transform_id()
    fake = ctypes.c_void_p(256)
    call = lambda obj, X=fake, M=fake, o=fake, f=fake, B=2, n=3, D=3, ldx=3, ws=None, wsb=0, sm=0: lib.evok_eval_transform_batched(  # noqa: E731
        obj, X, 0, ldx, M, sm, o, 0, B, n, D, 1, 0, ws, wsb, f, None)
    assert call(tid, X=None) == -1 and call(tid, M=None) == -1 and call(tid, o=None) == -1 and call(tid, f=None) == -1
    assert call(0) == -3 and call(5) == -3
    assert call(tid, D=0) == -2 and call(tid, ldx=2) == -2 and call(tid, B=-1) == -2 and call(tid, sm=-1) == -2
    assert call(1) == -7  # a built-in objective has no transformed family
    plain = FusedObjective("abi_plain", sums={"s": "x**2"}, value="s")
    assert call(plain.evok_objective_id) == -7
    assert call(tid, B=0) == 0 and call(tid, n=0) == 0  # nothing to evaluate: no launch
    # registration: the kernel count of the fourth family
    out = ctypes.c_int()
    names = (ctypes.c_char_p * 4)(*[b"k"] * 4)
    assert lib.evok_objective_register_transform(None, 1, names, 4, ctypes.byref(out)) == -1
    assert lib.evok_objective_register_transform(b"x", 1, names, 3, ctypes.byref(out)) == -2
    assert lib.evok_objective_register_transform(b"x", 0, names, 4, ctypes.byref(out)) == -2
    # workspace: none on the fused path, x - o, y and the GEMM's on the other
    assert lib.evok_eval_transform_workspace_bytes(fake, 0, 10, 16, 40) == 0
    big = lib.evok_eval_transform_workspace_bytes(fake, 0, 10, 16, 1000)
    assert big >= 2 * 10 * 16 * 1000 * 4
    # items chunked so that x - o and y stay within 256 MB
    assert lib.evok_eval_transform_workspace_bytes(fake, 0, 100000, 1000, 1000) <= (256 << 20) + (64 << 20)
