"""Run-time compiled objectives: a function of reductions over the elements or neighbour pairs of a row, given as Python
expressions, becomes an accumulator of the fused sampler (csrc/evok_sampler.cuh), compiled with NVRTC for sm_90a and
registered with libevok.so.

    f(x) = value(S_1, ..., S_k, D),    k <= 4,
    S_i = R_{j=0}^{D-1} term_i(x_j, j, D)              (an element term), or
    S_i = R_{j=0}^{D-2} term_i(x_j, x_{j+1}, j, D)     (a pair term: one that uses xn; empty when D = 1)

where the reduction R is a sum (`sums`), a product (`prods`), a maximum (`maxs`) or a minimum (`mins`); the k reductions share
one namespace.  An empty reduction is 0, 1, -inf or +inf respectively.  A NaN term makes its product, maximum or minimum NaN, as
torch.prod / amax / amin do (the kernels' max / min propagate NaN; fmaxf / fminf would not); +-inf pass through.

Pair terms give the chained test functions, e.g. Rosenbrock: {"s": "100*(xn - x**2)**2 + (1 - x)**2"}, value "s".  One
objective may mix both kinds.

`running` defines up to 2 running sums c_j = sum_{k<=j} h(x_k, k, D), inclusive of column j, with h an element term (x, j, D and
data; no xn, no running or reduction name).  A running name is usable in the element terms of every reduction, and nowhere
else (pair terms, running terms, `value`): Schwefel 1.2 is running {"c": "x"}, sums {"s": "c**2"}, value "s".  The kernels
compute c_j with one warp scan per step of 128 columns and a carry per row (fold_running in csrc/evok_sampler.cuh); the torch
function with cumsum.

One parse of the expressions gives both the CUDA accumulator and a torch function of the same formula (the evaluation of
CPU problems, other dtypes, rng="torch" and before-eval hooks; the float64 reference of the tests).

The expression language (anything else raises ValueError):
  - operators  + - * /, unary -, ** (an integer literal exponent expands to products, any other exponent is powf / torch.pow);
  - functions  abs sqrt exp log sin cos tan tanh floor minimum maximum  (minimum / maximum return the other operand when
    one is NaN, like fminf / fmaxf and torch.fmin / torch.fmax);
  - where(cond, a, b)  a conditional, CUDA (cond) ? a : b and torch.where; cond is one comparison < <= > >= == != of two
    expressions, and comparisons are allowed nowhere else.  As in IEEE arithmetic a comparison with NaN is false, except !=,
    which is true (CUDA and torch agree);
  - noise      rand() (uniform on [0, 1)) and randn() (standard normal), each occurrence its own independent draw: one per
    row and column in the element terms of sums, prods, maxs and mins, one per row in `value`, also inside where(...); not in a
    pair term or a running term, and without arguments.  At most 4 occurrences in the element terms and 4 in `value`; each
    element occurrence costs one Philox4x32-10 call per 4 columns and row.  The kernels draw from the Philox key of the
    population's own draw (csrc/evok_sampler.cuh: noise_bits), the torch function with torch.rand / torch.randn: the same
    distributions, not the same bits (as rng="torch").  Only a call draws: `rand` and `randn` remain usable as the names of
    reductions, running sums and data;
  - constants  pi, e, numeric literals;
  - names      x (the element), xn (the next element x_{j+1}), j (the 0-based column of x) and D (the row length) in a
    term, and the running names in an element term of a reduction; the reduction names and D in `value`.  With a transform
    (`transform=True` here, the matrix and offset bound by FusedObjective) also y, entry j of the transformed row
    y = M (x - o), in element and running terms, and yn = y_{j+1} in pair terms (a term that uses xn or yn is a pair term).
  - data       up to 4 more names, each bound to a float32 tensor (`data={"t": t, "lam": lam}`).  Last dimension 1 makes a
    scalar, usable in the terms and in `value`; any other last dimension makes a vector, which must have the row length D and is
    usable in the terms only: `t` is its entry at column j and, in a pair term, `t_n` its entry at column j + 1 (as x and xn).
    Leading dimensions are batch dimensions: one data set per item of a batched search.
The CUDA side evaluates in float32 with the precise libdevice functions (no fast math) and contracts a * b + c into fma.
The source of an objective without pair terms is exactly that of the element-only language (no pair code in it), the source
of one without data is exactly that of the language without data, and the source of one of sums without running sums is exactly
that of the language before products, maxima, minima and running sums.  The source of an objective without a transform is
exactly that of the language without transforms; one with a transform declares kTransform and its folds take y after x.  Which data name is a scalar and which a vector is part of
the source; the tensors are not: they are bound to an instance of the compiled objective (`bind_instance`) and reach the
kernels as a launch argument, so objectives with the same expressions and kinds share one compilation whatever their data.
"""

from __future__ import annotations

import ast
import ctypes
import math
import os
import re
import threading
from ctypes import c_char_p, c_int, c_size_t, c_void_p
from typing import Callable, Dict, Optional

import numpy as np
import torch

from . import _native as nat

_PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_PKG, "csrc")
INCLUDE = os.path.join(os.path.dirname(_PKG), "include")

MAX_SUMS = 4  # reductions of all kinds together
MAX_RUNNING = 2
MAX_DATA = 4  # EVOK_MAX_DATA
MAX_INT_POWER = 16

FUNCTIONS = {
    "abs": ("fabsf", torch.abs), "sqrt": ("sqrtf", torch.sqrt), "exp": ("expf", torch.exp), "log": ("logf", torch.log),
    "sin": ("sinf", torch.sin), "cos": ("cosf", torch.cos), "tan": ("tanf", torch.tan), "tanh": ("tanhf", torch.tanh),
    "floor": ("floorf", torch.floor), "minimum": ("fminf", torch.fmin), "maximum": ("fmaxf", torch.fmax),
}
CONSTANTS = {"pi": math.pi, "e": math.e}
NOISE = {"rand": torch.rand, "randn": torch.randn}  # zero-argument functions: one independent draw per occurrence
MAX_DRAWS = 4  # occurrences of rand() / randn() in the element terms, and again in `value`
_ARITY = {"minimum": 2, "maximum": 2}
_BINOPS = {ast.Add: "+", ast.Sub: "-", ast.Mult: "*", ast.Div: "/"}
_COMPARE = {ast.Lt: ("<", torch.lt), ast.LtE: ("<=", torch.le), ast.Gt: (">", torch.gt), ast.GtE: (">=", torch.ge),
            ast.Eq: ("==", torch.eq), ast.NotEq: ("!=", torch.ne)}
_ALLOWED_TEXT = ("allowed: + - * / ** and unary -, the functions " + " ".join(FUNCTIONS) + ", where(cond, a, b) with one comparison "
                 "< <= > >= == != as cond, the constants pi and e, numeric literals and the names {names}")


def _float_literal(v: float) -> str:
    with np.errstate(over="ignore"):
        f = float(np.float32(v))
    if not math.isfinite(f):
        raise ValueError(f"the literal {v!r} is not a finite float32")
    return repr(f) + "f"


class _Expr:
    """One translated expression: `cuda` is its CUDA text over the given identifiers, `torch(env)` evaluates it on tensors and
    `names` holds the Python names whose identifiers `cuda` contains."""

    def __init__(self, cuda: str, fn: Callable, names: frozenset = frozenset()):
        self.cuda, self.torch, self.names = cuda, fn, names


def _as_tensor(v, env):
    return v if isinstance(v, torch.Tensor) else torch.as_tensor(v, dtype=env["_dtype"], device=env["_device"])


def _int_exponent(node) -> Optional[int]:
    """The integer value of a literal exponent (2, -3, 2.0), else None."""
    sign = 1
    if isinstance(node, ast.UnaryOp) and isinstance(node.op, (ast.USub, ast.UAdd)):
        sign = -1 if isinstance(node.op, ast.USub) else 1
        node = node.operand
    if isinstance(node, ast.Constant) and type(node.value) in (int, float) and float(node.value).is_integer():
        n = sign * int(node.value)
        return n if abs(n) <= MAX_INT_POWER else None
    return None


def _translate(node, names: Dict[str, str], where: str, draws: Optional["_Draws"] = None) -> _Expr:
    """node: a tree of `_parse`; names: the Python names allowed here -> their CUDA identifiers; draws: where rand() / randn() here
    draw from (None: they are refused here)."""
    allowed = _ALLOWED_TEXT.format(names=", ".join(names))
    if isinstance(node, ast.Expression):
        return _translate(node.body, names, where, draws)
    if isinstance(node, ast.Constant):
        if type(node.value) not in (int, float):
            raise ValueError(f"{where}: the literal {node.value!r} is not a number; {allowed}")
        v = float(node.value)
        return _Expr(_float_literal(v), lambda env, v=v: v)
    if isinstance(node, ast.Name):
        if node.id in names:
            return _Expr(names[node.id], lambda env, n=node.id: env[n], frozenset((node.id,)))
        if node.id in CONSTANTS:
            v = CONSTANTS[node.id]
            return _Expr(_float_literal(v), lambda env, v=v: v)
        raise ValueError(f"{where}: unknown name {node.id!r}; {allowed}")
    if isinstance(node, ast.UnaryOp):
        a = _translate(node.operand, names, where, draws)
        if isinstance(node.op, ast.USub):
            return _Expr(f"(-{a.cuda})", lambda env: -a.torch(env), a.names)
        if isinstance(node.op, ast.UAdd):
            return a
        raise ValueError(f"{where}: the operator {type(node.op).__name__} is not supported; {allowed}")
    if isinstance(node, ast.BinOp):
        a = _translate(node.left, names, where, draws)
        if isinstance(node.op, ast.Pow):
            n = _int_exponent(node.right)
            if n is not None:
                if n == 0:
                    return _Expr("1.0f", lambda env: 1.0)
                prod = "(" + " * ".join([a.cuda] * abs(n)) + ")"
                return _Expr(prod if n > 0 else f"(1.0f / {prod})", lambda env: a.torch(env) ** n, a.names)
            b = _translate(node.right, names, where, draws)
            return _Expr(f"powf({a.cuda}, {b.cuda})", lambda env: torch.pow(_as_tensor(a.torch(env), env), b.torch(env)), a.names | b.names)
        if type(node.op) not in _BINOPS:
            raise ValueError(f"{where}: the operator {type(node.op).__name__} is not supported; {allowed}")
        b = _translate(node.right, names, where, draws)
        op = _BINOPS[type(node.op)]
        fn = {"+": lambda env: a.torch(env) + b.torch(env), "-": lambda env: a.torch(env) - b.torch(env),
              "*": lambda env: a.torch(env) * b.torch(env), "/": lambda env: a.torch(env) / b.torch(env)}[op]
        return _Expr(f"({a.cuda} {op} {b.cuda})", fn, a.names | b.names)
    if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id in NOISE:
        if node.args or node.keywords:
            raise ValueError(f"{where}: {node.func.id}() takes no arguments, got {ast.unparse(node)!r}")
        if draws is None:
            raise ValueError(f"{where}: {node.func.id}() draws noise, which is allowed in the element terms of sums, prods, maxs and mins "
                             f"and in `value` only (not in a pair term or a running term)")
        return draws.take(node.func.id, where)
    if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "where":
        if node.keywords or len(node.args) != 3:
            raise ValueError(f"{where}: where takes 3 positional arguments (cond, a, b), got {ast.unparse(node)!r}")
        cond = node.args[0]
        if not (isinstance(cond, ast.Compare) and len(cond.ops) == 1 and type(cond.ops[0]) in _COMPARE):
            raise ValueError(f"{where}: the condition of where must be one comparison < <= > >= == != of two expressions, got "
                             f"{ast.unparse(cond)!r}")
        op, top = _COMPARE[type(cond.ops[0])]
        l, r = _translate(cond.left, names, where, draws), _translate(cond.comparators[0], names, where, draws)
        a, b = _translate(node.args[1], names, where, draws), _translate(node.args[2], names, where, draws)

        def where_fn(env):
            lv, rv = _as_tensor(l.torch(env), env), _as_tensor(r.torch(env), env)
            return torch.where(top(lv, rv), _as_tensor(a.torch(env), env), _as_tensor(b.torch(env), env))

        return _Expr(f"(({l.cuda} {op} {r.cuda}) ? {a.cuda} : {b.cuda})", where_fn, l.names | r.names | a.names | b.names)
    if isinstance(node, ast.Compare):
        raise ValueError(f"{where}: Compare ({ast.unparse(node)!r}) is not supported outside where: a comparison is allowed only as "
                         f"the condition of where(cond, a, b); {allowed}")
    if isinstance(node, ast.Call):
        if not isinstance(node.func, ast.Name) or node.func.id not in FUNCTIONS:
            what = node.func.id if isinstance(node.func, ast.Name) else ast.unparse(node.func)
            raise ValueError(f"{where}: the function {what!r} is not supported; {allowed}")
        if node.keywords:
            raise ValueError(f"{where}: keyword arguments are not supported; {allowed}")
        name = node.func.id
        arity = _ARITY.get(name, 1)
        if len(node.args) != arity:
            raise ValueError(f"{where}: {name} takes {arity} argument(s), got {len(node.args)}")
        args = [_translate(a, names, where, draws) for a in node.args]
        cname, tfn = FUNCTIONS[name]
        return _Expr(f"{cname}(" + ", ".join(a.cuda for a in args) + ")",
                     lambda env: tfn(*[_as_tensor(a.torch(env), env) for a in args]), frozenset().union(*(a.names for a in args)))
    raise ValueError(f"{where}: {type(node).__name__} ({ast.unparse(node)!r}) is not supported; {allowed}")


def _parse(text: str, where: str):
    """The tree of an expression, for `_translate`, and the names it reads (not the functions it calls: a reduction, running sum
    or data name may be `rand`)."""
    if not isinstance(text, str):
        raise ValueError(f"{where}: expected an expression string, got {type(text).__name__}")
    try:
        tree = ast.parse(text, mode="eval")
    except SyntaxError as e:
        raise ValueError(f"{where}: not a Python expression: {text!r} ({e.msg})") from None
    called, reads = set(), set()
    for n in ast.walk(tree):  # breadth first: a call comes before the name it calls
        if isinstance(n, ast.Call):
            called.add(id(n.func))
        elif isinstance(n, ast.Name) and id(n) not in called:
            reads.add(n.id)
    return tree, reads


class _Draws:
    """The occurrences of rand() / randn() in one context (the element terms, or `value`), in source order: occurrence k is
    `cuda(k, name)` in the CUDA source and a fresh torch.rand / torch.randn of the context's shape (env["_shape"]) in torch."""

    def __init__(self, context: str, cuda: Callable[[int, str], str]):
        self.context, self.cuda, self.normal = context, cuda, []

    def take(self, name: str, where: str) -> _Expr:
        if len(self.normal) >= MAX_DRAWS:
            raise ValueError(f"{where}: at most {MAX_DRAWS} occurrences of rand() / randn() in {self.context}, got more")
        k = len(self.normal)
        self.normal.append(name == "randn")
        fn = NOISE[name]
        return _Expr(self.cuda(k, name), lambda env: fn(env["_shape"], dtype=env["_dtype"], device=env["_device"]))

    @property
    def normal_mask(self) -> int:
        return sum(1 << k for k, n in enumerate(self.normal) if n)


# the reductions in slot order, with their keyword, the identity their slot starts from and their warp butterfly
REDUCTIONS = ("sum", "prod", "max", "min")
GROUP_OF = {"sum": "sums", "prod": "prods", "max": "maxs", "min": "mins"}
IDENTITY = {"sum": "0.f", "prod": "1.f", "max": "-evok::inf()", "min": "evok::inf()"}
WARP_REDUCE = {"sum": "warp_sum", "prod": "warp_prod", "max": "warp_max", "min": "warp_min"}

_RESERVED = {"x", "j", "D"} | set(CONSTANTS) | set(FUNCTIONS)
_RESERVED_DATA = _RESERVED | {"xn"}


def data_kinds(data: dict) -> Dict[str, bool]:
    """{name: is a vector} of a `data` dict of tensors, after the checks on the names and tensors (ValueError)."""
    if not isinstance(data, dict) or len(data) > MAX_DATA:
        raise ValueError(f"data: expected a dict of at most {MAX_DATA} named float32 tensors")
    kinds = {}
    for name, t in data.items():
        if not (isinstance(name, str) and name.isidentifier()) or name in _RESERVED_DATA or name.endswith("_n"):
            raise ValueError(f"data: {name!r} cannot name data (a data name is an identifier that does not end in '_n', other than "
                             f"{sorted(_RESERVED_DATA)})")
        if not (isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.ndim >= 1 and t.shape[-1] >= 1):
            what = f"{tuple(t.shape)} {t.dtype}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"data[{name!r}]: expected a float32 tensor with at least one dimension, got {what}")
        kinds[name] = t.shape[-1] != 1
    return kinds


class ObjectiveSpec:
    """The parsed form of an objective: `source` is the CUDA translation unit, `torch_fn(X)` the torch function.  `reductions`
    maps every reduction name to its combine operation ("sum", "prod", "max" or "min") in slot order, `pairs` names the
    reductions whose term uses xn (reduced over the neighbour pairs of a row; the others over its elements) and `running` the
    running-sum terms."""

    def __init__(self, sums: Optional[Dict[str, str]], value: str, kinds: Optional[Dict[str, bool]] = None, *,
                 prods: Optional[Dict[str, str]] = None, maxs: Optional[Dict[str, str]] = None, mins: Optional[Dict[str, str]] = None,
                 running: Optional[Dict[str, str]] = None, transform: bool = False):
        """kinds: {data name: is a vector} in binding order (`data_kinds`), None or empty for an objective without data.
        transform: the terms may read y and yn, the entries of the transformed row (and at least one of them must)."""
        self.kinds = dict(kinds or {})
        self.transform = bool(transform)
        # the names of the next column's entries: a term that reads one is a pair term
        nexts = {"xn", "yn"} if self.transform else {"xn"}
        if value is None:
            raise ValueError("value: an objective needs a `value` expression of its reductions")
        groups = {"sums": sums, "prods": prods, "maxs": maxs, "mins": mins}
        for what, g in groups.items():
            if g is not None and not isinstance(g, dict):
                raise ValueError(f"{what}: expected a dict of named term expressions, got {type(g).__name__}")
        if prods is None and maxs is None and mins is None:
            if not isinstance(sums, dict) or not 1 <= len(sums) <= MAX_SUMS:
                raise ValueError(f"sums: expected a dict of 1 to {MAX_SUMS} named term expressions")
        elif not 1 <= sum(len(g or {}) for g in groups.values()) <= MAX_SUMS:
            raise ValueError(f"sums, prods, maxs, mins: expected 1 to {MAX_SUMS} reductions in all, got "
                             f"{sum(len(g or {}) for g in groups.values())}")
        self.reductions, texts = {}, {}
        for (what, g), op in zip(groups.items(), REDUCTIONS):
            for s, t in (g or {}).items():
                if not (isinstance(s, str) and s.isidentifier()) or s in _RESERVED:
                    raise ValueError(f"{what}: {s!r} cannot name a {op} (a reduction name is an identifier other than {sorted(_RESERVED)})")
                if s in self.reductions:
                    raise ValueError(f"{what}: {s!r} names two reductions; sums, prods, maxs and mins share one namespace")
                self.reductions[s], texts[s] = op, t
        if running is not None and not isinstance(running, dict) or len(running or {}) > MAX_RUNNING:
            raise ValueError(f"running: expected a dict of at most {MAX_RUNNING} named running-sum terms")
        running = dict(running or {})
        for c in running:
            if not (isinstance(c, str) and c.isidentifier()) or c in _RESERVED_DATA:
                raise ValueError(f"running: {c!r} cannot name a running sum (an identifier other than {sorted(_RESERVED_DATA)})")
            if c in self.reductions:
                raise ValueError(f"running: {c!r} is also the name of a reduction")
        self.sums, self.value = dict(sums or {}), value
        self.prods, self.maxs, self.mins, self.running = dict(prods or {}), dict(maxs or {}), dict(mins or {}), running
        term_names = {"x": "x", "xn": "xn", "j": "jf", "D": "Df"}
        if self.transform:
            taken = sorted({"y", "yn"} & (set(self.reductions) | set(running) | set(self.kinds)))
            if taken:
                raise ValueError(f"{taken[0]!r} names a reduction, running sum or data, but with a transform it is an entry of the "
                                 "transformed row y = M (x - o)")
            term_names.update(y="y", yn="yn")
        value_names = {s: f"S_{s}" for s in self.reductions}
        value_names["D"] = "Df"
        for name, vector in self.kinds.items():
            if name in self.reductions:
                raise ValueError(f"data: {name!r} is the name of a {self.reductions[name]}")
            if name in running:
                raise ValueError(f"data: {name!r} is the name of a running sum")
            # a vector's entries at columns j and j + 1, handed to add / add_pair; a scalar is a member of the accumulator
            term_names.update({name: f"v_{name}", f"{name}_n": f"vn_{name}"} if vector else {name: f"c_{name}"})
            if not vector:
                value_names[name] = f"c_{name}"
        allowed_where = ("a running sum is usable in the element terms of sums, prods, maxs and mins only (not in a pair term, a "
                         "running term or `value`)")
        vectors = [n for n, v in self.kinds.items() if v]

        def next_entry(e: _Expr) -> Optional[str]:  # a vector whose entry at column j + 1 (name_n) the expression reads
            return next((n for n in vectors if f"{n}_n" in e.names), None)

        running_trees = {c: _parse(t, f"running[{c!r}]") for c, t in running.items()}
        for c, (_, used) in running_trees.items():
            self._check_data_names(used, f"running[{c!r}]", term=True)
            bad = used & (set(running) | set(self.reductions))
            if bad:
                raise ValueError(f"running[{c!r}]: {sorted(bad)[0]!r}: a running term is an element term of x, j, D and data; "
                                 f"{allowed_where}")
        # noise: element occurrences are the column entries d[kVectors + k] (after the data vectors'), occurrences in `value` the
        # row's draws in finish (evok_sampler.cuh: DataCols::draw4, value_rand / value_randn)
        self.element_draws = _Draws("the element terms", lambda k, name: f"d[{len(vectors) + k}]")
        self.value_draws = _Draws("`value`", lambda k, name: f"evok::value_{name}(key, sw, row, {MAX_DRAWS + k})")
        self.running_terms = {c: _translate(tree, {k: v for k, v in term_names.items() if k not in nexts}, f"running[{c!r}]")
                              for c, (tree, _) in running_trees.items()}
        for c, e in self.running_terms.items():
            n = next_entry(e)
            if n:
                raise ValueError(f"running[{c!r}]: {n}_n is the entry at column j + 1, which only a pair term has")
        run_names = dict(term_names, **{c: f"r[{i}]" for i, c in enumerate(running)})
        term_trees = {s: _parse(t, f"{GROUP_OF[self.reductions[s]]}[{s!r}]") for s, t in texts.items()}
        for s, (_, used) in term_trees.items():
            self._check_data_names(used, f"{GROUP_OF[self.reductions[s]]}[{s!r}]", term=True)
            if used & set(running) and used & nexts:
                raise ValueError(f"{GROUP_OF[self.reductions[s]]}[{s!r}]: {sorted(used & set(running))[0]!r} in a pair term; "
                                 f"{allowed_where}")
        value_tree, used = _parse(value, "value")
        self._check_data_names(used, "value", term=False)
        if used & set(running):
            raise ValueError(f"value: {sorted(used & set(running))[0]!r} is a running sum; {allowed_where}")
        # a term that reads xn (or yn) is a pair term, where rand() / randn() are refused
        self.terms = {s: _translate(tree, run_names, f"{GROUP_OF[self.reductions[s]]}[{s!r}]", None if used & nexts else self.element_draws)
                      for s, (tree, used) in term_trees.items()}
        self.pairs = frozenset(s for s, e in self.terms.items() if e.names & nexts)
        if self.transform and not any(e.names & {"y", "yn"} for e in list(self.terms.values()) + list(self.running_terms.values())):
            raise ValueError("transform: no term reads y or yn, the entries of the transformed row; an objective of x alone needs no "
                             "transform")
        for s, e in self.terms.items():
            n = next_entry(e)
            if n and s not in self.pairs:
                raise ValueError(f"{GROUP_OF[self.reductions[s]]}[{s!r}]: {n}_n is the entry of {n!r} at column j + 1, "
                                 f"which only a pair term (one that uses xn) has; an element term uses {n!r}")
        self.value_expr = _translate(value_tree, value_names, "value", self.value_draws)
        self.noisy = bool(self.element_draws.normal or self.value_draws.normal)
        self.source = self._cuda_source()

    def _check_data_names(self, used: set, where: str, term: bool) -> None:
        for name, vector in self.kinds.items():
            if not vector and f"{name}_n" in used:
                raise ValueError(f"{where}: {name}_n: {name!r} is a scalar (its last dimension is 1) and has no next entry; use {name!r}")
            if vector and not term and (name in used or f"{name}_n" in used):
                raise ValueError(f"{where}: {name!r} is a vector with one entry per column; it can be used in the terms of `sums` only")

    def _cuda_source(self) -> str:
        k = range(len(self.terms))
        uses_j = lambda es: any("j" in e.names for e in es)  # noqa: E731
        element = [(i, e) for i, (s, e) in zip(k, self.terms.items()) if s not in self.pairs]
        pair = [(i, e) for i, (s, e) in zip(k, self.terms.items()) if s in self.pairs]
        ops = [self.reductions[s] for s in self.terms]
        nr = len(self.running_terms)
        # data: slot i of the binding is data name i; the vectors are numbered among themselves in the same order
        vectors = [n for n, v in self.kinds.items() if v]
        nd = len(self.element_draws.normal)
        nv = max(len(vectors) + nd, 1)  # the column entries of a fold: data vectors, then element draws

        def entries(es, prefix, array, suffix=""):  # the locals of the vector entries that the terms `es` read (name + suffix)
            return [f"    const float {prefix}_{n} = {array}[{i}];" for i, n in enumerate(vectors) if any(n + suffix in e.names for _, e in es)]

        def combine(i, e):  # slot i folds the term e with its reduction's operation
            return {"sum": f"    s{i} += {e};", "prod": f"    s{i} *= {e};", "max": f"    s{i} = evok::max_nan(s{i}, {e});",
                    "min": f"    s{i} = evok::min_nan(s{i}, {e});"}[ops[i]]

        lines = ['#include "evok_sampler.cuh"', "", "namespace evok_user {", "struct Acc {"]
        if self.transform:
            lines.append("  static constexpr bool kTransform = true;")
        # the column values a fold takes: x, or x and its transformed entry y
        col = "float x, float y, " if self.transform else "float x, "
        cols = "float x, float xn, float y, float yn, " if self.transform else "float x, float xn, "
        if pair:
            lines.append("  static constexpr bool kPairs = true;")
        if nr:
            lines.append("  static constexpr bool kRunning = true;")
            lines.append(f"  static constexpr int kRunningSums = {nr};")
        if self.kinds:
            lines.append("  static constexpr bool kData = true;")
            lines.append(f"  static constexpr int kVectors = {len(vectors)};")
        if self.noisy:
            lines.append("  static constexpr bool kNoise = true;")
            lines.append(f"  static constexpr int kDraws = {nd};")
            lines.append(f"  static constexpr unsigned kNormalDraws = {self.element_draws.normal_mask}u;")
        lines.append("  float Df;")
        lines.append("  float " + ", ".join(f"s{i} = {IDENTITY[ops[i]]}" for i in k) + ";")
        data_arg = f"const float (&d)[{nv}], " if self.kinds or nd else ""
        if self.kinds:
            slot = {n: i for i, n in enumerate(self.kinds)}
            lines.append(f"  const float* vec[{nv}];")
            scalars = [n for n, v in self.kinds.items() if not v]
            if scalars:
                lines.append("  float " + ", ".join(f"c_{n}" for n in scalars) + ";")
            init = ["Df((float)D)", "vec{" + ", ".join(f"b.p[{slot[n]}]" for n in vectors) + "}"]
            init += [f"c_{n}(__ldg(b.p[{slot[n]}]))" for n in scalars]
            lines.append("  __device__ __forceinline__ Acc(int64_t D, const evok::DataBinding& b) : " + ", ".join(init) + " {}")
        else:
            lines.append("  __device__ __forceinline__ explicit Acc(int64_t D) : Df((float)D) {}")
        if nr:
            run = [(i, e) for i, e in enumerate(self.running_terms.values())]
            lines.append(f"  __device__ __forceinline__ void running({col}int64_t j, {data_arg}float (&h)[{nr}]) {{")
            if uses_j(e for _, e in run):
                lines.append("    const float jf = (float)j;")
            lines += entries(run, "v", "d")
            lines += [f"    h[{i}] = {e.cuda};" for i, e in run]
            lines.append("  }")
            lines.append(f"  __device__ __forceinline__ void add({col}int64_t j, {data_arg}const float (&r)[{nr}]) {{")
        elif data_arg:
            lines.append(f"  __device__ __forceinline__ void add({col}int64_t j, const float (&d)[{nv}]) {{")
        else:
            lines.append(f"  __device__ __forceinline__ void add({col}int64_t j) {{")
        if uses_j(e for _, e in element):
            lines.append("    const float jf = (float)j;")
        lines += entries(element, "v", "d")
        lines += [combine(i, e.cuda) for i, e in element]
        lines.append("  }")
        if pair:
            if data_arg:
                lines.append(f"  __device__ __forceinline__ void add_pair({cols}int64_t j, const float (&d)[{nv}], "
                             f"const float (&dn)[{nv}]) {{")
            else:
                lines.append(f"  __device__ __forceinline__ void add_pair({cols}int64_t j) {{")
            if uses_j(e for _, e in pair):
                lines.append("    const float jf = (float)j;")
            lines += entries(pair, "v", "d") + entries(pair, "vn", "dn", "_n")
            lines += [combine(i, e.cuda) for i, e in pair]
            lines.append("  }")
        if self.noisy:
            lines.append("  __device__ __forceinline__ float finish(int64_t, const evok::PhiloxKey& key, uint32_t sw, uint64_t row) {")
        else:
            lines.append("  __device__ __forceinline__ float finish(int64_t) {")
        lines += [f"    const float S_{s} = evok::{WARP_REDUCE[ops[i]]}(s{i});" for i, s in zip(k, self.terms)]
        lines.append(f"    return {self.value_expr.cuda};")
        lines += ["  }", "};", "}  // namespace evok_user", ""]
        return "\n".join(lines)

    def torch_fn(self, X: torch.Tensor, data: Optional[Dict[str, torch.Tensor]] = None, transform: Optional[tuple] = None) -> torch.Tensor:
        """The fitnesses of the rows of X (..., N, D).  data: the tensors of the data names, cast to X's dtype and device; their
        leading (batch) dimensions broadcast against the batch dimensions of X, and the result has the broadcast shape.
        transform: (M (..., D, D), o (..., D)) of an objective with a transform, cast likewise: y = (X - o) M^T with torch.matmul,
        their batch dimensions broadcast as the data's do."""
        D = X.shape[-1]
        Dt = torch.tensor(float(D), dtype=X.dtype, device=X.device)
        env = {"x": X, "j": torch.arange(D, dtype=X.dtype, device=X.device), "D": Dt, "_dtype": X.dtype, "_device": X.device}
        # a pair term on (x_j, x_{j+1}) for j = 0 .. D-2: an empty reduction when D = 1
        penv = {"x": X[..., :-1], "xn": X[..., 1:], "j": torch.arange(max(D - 1, 0), dtype=X.dtype, device=X.device), "D": Dt,
                "_dtype": X.dtype, "_device": X.device}
        venv = {}
        rows = X.shape[:-1]  # the shape of the result
        if self.kinds:
            check_data(self.kinds, data, D)
            for name, vector in self.kinds.items():
                t = data[name].to(dtype=X.dtype, device=X.device)
                rows = torch.broadcast_shapes(rows, tuple(t.shape[:-1]) + (1,))
                t = t.unsqueeze(-2)  # (*batch, 1, D or 1) against the rows (*batch, N, D)
                env[name] = t
                penv[name] = t[..., :-1] if vector else t
                if vector:
                    penv[f"{name}_n"] = t[..., 1:]
                else:
                    venv[name] = t[..., 0]
        if self.transform:
            if transform is None:
                raise ValueError("transform: this objective reads the transformed row y = M (x - o); expected (M, o)")
            M, o = (t.to(dtype=X.dtype, device=X.device) for t in transform)
            Y = torch.matmul(X - o.unsqueeze(-2), M.mT)
            rows = torch.broadcast_shapes(rows, Y.shape[:-1])
            env["y"], penv["y"], penv["yn"] = Y, Y[..., :-1], Y[..., 1:]
        env["_shape"] = rows + (D,)  # of an element draw (rand() / randn() in an element term): one per row and column
        for c, e in self.running_terms.items():  # c_j = sum_{k <= j} h(x_k, k, D)
            env[c] = torch.broadcast_to(_as_tensor(e.torch(env), env), rows + (D,)).cumsum(dim=-1)
        for s, e in self.terms.items():
            en = penv if s in self.pairs else env
            shape = rows + (en["x"].shape[-1],)
            t = torch.broadcast_to(_as_tensor(e.torch(en), en), shape)
            op = self.reductions[s]
            if op == "sum":
                venv[s] = t.sum(dim=-1)
            elif op == "prod":
                venv[s] = t.prod(dim=-1)
            elif shape[-1] == 0:  # torch.amax / amin refuse an empty dimension: the identity
                venv[s] = torch.full(rows, -math.inf if op == "max" else math.inf, dtype=t.dtype, device=t.device)
            else:
                venv[s] = t.amax(dim=-1) if op == "max" else t.amin(dim=-1)
        venv.update(D=Dt, _dtype=X.dtype, _device=X.device, _shape=rows)
        return torch.broadcast_to(_as_tensor(self.value_expr.torch(venv), venv), rows)


def check_data(kinds: Dict[str, bool], data: Optional[Dict[str, torch.Tensor]], D: int) -> None:
    """ValueError unless `data` holds a tensor of the declared kind for every name, with every vector of length D."""
    if data is None or list(data) != list(kinds):
        raise ValueError(f"data: expected tensors for the names {list(kinds)}, got {None if data is None else list(data)}")
    for name, vector in kinds.items():
        n = data[name].shape[-1]
        if (n != 1) != vector:
            raise ValueError(f"data[{name!r}]: a {'vector' if vector else 'scalar'} in the expressions, but its last dimension is {n}")
        if vector and n != D:
            raise ValueError(f"data[{name!r}]: the vector has length {n}, the rows have length {D}")


# ------------------------------------------------------------------------------------------------ NVRTC
def kernel_expressions() -> list:
    """The 22 kernels of a registered objective, in the EVOK_OBJ_KERNEL_* order of include/evok.h (kernel_index in
    csrc/evok_sample_eval.cu computes the same positions)."""
    b = lambda v: "true" if v else "false"  # noqa: E731
    out = []
    for push in (False, True):  # EVOK_OBJ_KERNEL_SAMPLE, EVOK_OBJ_KERNEL_PUSH: + 4 sym + 2 store + vec
        for sym in (False, True):
            for store in (False, True):
                for vec in (False, True):
                    out.append(f"evok::sample_eval_kernel<evok_user::Acc, {b(sym)}, {b(store)}, {b(vec)}, {b(push)}, false>")
    for store in (False, True):  # EVOK_OBJ_KERNEL_SQ: + 2 store + vec
        for vec in (False, True):
            out.append(f"evok::sample_eval_kernel<evok_user::Acc, false, {b(store)}, {b(vec)}, false, true>")
    for vec in (False, True):  # EVOK_OBJ_KERNEL_EVAL: + vec
        out.append(f"evok::eval_kernel<evok_user::Acc, {b(vec)}>")
    return out


def batched_kernel_expressions() -> list:
    """The 8 batched samplers of a registered objective, in the order of EVOK_OBJ_KERNEL_BATCHED + 4 sym + 2 store + vec of
    include/evok.h (kernel_index in csrc/evok_sample_eval.cu computes the same positions).  They are compiled from the same
    source as `kernel_expressions`, as a second image, on the first batched use (`compile_batched`)."""
    b = lambda v: "true" if v else "false"  # noqa: E731
    return [f"evok::sample_eval_batched_kernel<evok_user::Acc, {b(sym)}, {b(store)}, {b(vec)}>"
            for sym in (False, True) for store in (False, True) for vec in (False, True)]


def eval_batched_kernel_expressions() -> list:
    """The 2 batched evaluation kernels of a registered objective, in the order of EVOK_OBJ_KERNEL_EVAL_BATCHED + vec of
    include/evok.h.  They are compiled from the same source as `kernel_expressions`, as a third image, on the first batched
    evaluation (`compile_eval_batched`)."""
    return [f"evok::eval_batched_kernel<evok_user::Acc, {'true' if vec else 'false'}>" for vec in (False, True)]


def transform_kernel_expressions() -> list:
    """The 4 kernels of an objective with a transform, in the order of EVOK_OBJ_KERNEL_TRANSFORM (+ vec, then + 2 + vec) of
    include/evok.h: the fused small-D evaluation and the evaluation behind the GEMM.  They are its only kernels: no sampler can
    produce the transformed row one column group at a time."""
    b = lambda v: "true" if v else "false"  # noqa: E731
    return ([f"evok::eval_transform_fused_kernel<evok_user::Acc, {b(vec)}>" for vec in (False, True)]
            + [f"evok::eval_transform_kernel<evok_user::Acc, {b(vec)}>" for vec in (False, True)])


N_KERNELS = 22
N_BATCHED_KERNELS = 8
N_EVAL_BATCHED_KERNELS = 2
N_TRANSFORM_KERNELS = 4
# -default-device: the declarations of the C ABI in include/evok.h (reached through evok_sampler.cuh) are unannotated
NVRTC_OPTIONS = ("--gpu-architecture=sm_90a", "-std=c++17", "--fmad=true", "--ptxas-options=-v", "-default-device", f"-I{CSRC}",
                 f"-I{INCLUDE}")

_nvrtc: Optional[ctypes.CDLL] = None


def _nvrtc_candidates() -> list:
    cands = []
    try:
        import nvidia.cuda_nvrtc as m  # the NVRTC wheel torch depends on

        for d in m.__path__:
            cands += sorted((os.path.join(d, "lib", f) for f in os.listdir(os.path.join(d, "lib")) if re.fullmatch(r"libnvrtc\.so\.\d+", f)),
                            reverse=True)
    except (ImportError, OSError):
        pass
    from torch.utils.cpp_extension import CUDA_HOME

    for home in (CUDA_HOME, "/usr/local/cuda"):
        if home:
            cands.append(os.path.join(home, "lib64", "libnvrtc.so"))
    return cands


def nvrtc() -> ctypes.CDLL:
    global _nvrtc
    if _nvrtc is None:
        for path in _nvrtc_candidates():
            if os.path.exists(path):
                _nvrtc = ctypes.CDLL(path)
                break
        else:
            raise RuntimeError("NVRTC not found: a fused objective is compiled with the libnvrtc of torch's nvidia-cuda-nvrtc wheel or "
                               "of the CUDA toolkit")
        P = ctypes.POINTER
        for name, res, args in (
            ("nvrtcCreateProgram", c_int, [P(c_void_p), c_char_p, c_char_p, c_int, c_void_p, c_void_p]),
            ("nvrtcAddNameExpression", c_int, [c_void_p, c_char_p]),
            ("nvrtcCompileProgram", c_int, [c_void_p, c_int, P(c_char_p)]),
            ("nvrtcGetLoweredName", c_int, [c_void_p, c_char_p, P(c_char_p)]),
            ("nvrtcGetProgramLogSize", c_int, [c_void_p, P(c_size_t)]),
            ("nvrtcGetProgramLog", c_int, [c_void_p, c_char_p]),
            ("nvrtcGetCUBINSize", c_int, [c_void_p, P(c_size_t)]),
            ("nvrtcGetCUBIN", c_int, [c_void_p, c_char_p]),
            ("nvrtcDestroyProgram", c_int, [P(c_void_p)]),
            ("nvrtcGetErrorString", c_char_p, [c_int]),
        ):
            fn = getattr(_nvrtc, name)
            fn.restype, fn.argtypes = res, args
    return _nvrtc


class CompiledObjective:
    """An NVRTC compilation of one generated source: the cubin, the lowered kernel names, the ptxas info per kernel
    ({expression: {"registers", "spill_stores", "spill_loads", "stack"}}), the compile wall time and, once registered, the id."""

    def __init__(self, cubin: bytes, names: list, kernel_info: dict, seconds: float):
        self.cubin, self.names, self.kernel_info, self.seconds = cubin, names, kernel_info, seconds
        self.objective_id: Optional[int] = None


def _ptxas_info(log: str, lowered: Dict[str, str]) -> dict:
    by_lowered = {v: k for k, v in lowered.items()}
    info, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = by_lowered.get(m.group(1))
            if cur is not None:
                info[cur] = {}
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            info[cur].update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            info[cur]["registers"] = int(m.group(1))
    return info


def compile_source(source: str, expressions: Optional[list] = None) -> CompiledObjective:
    """Compile `source` with NVRTC for sm_90a and lower the names of `expressions` (default: the 22 objective kernels)."""
    import time

    lib = nvrtc()
    expressions = kernel_expressions() if expressions is None else expressions
    t0 = time.perf_counter()
    prog = c_void_p()

    def ok(rc, what):
        if rc != 0:
            raise RuntimeError(f"{what}: {lib.nvrtcGetErrorString(rc).decode()}")

    ok(lib.nvrtcCreateProgram(ctypes.byref(prog), source.encode(), b"evok_objective.cu", 0, None, None), "nvrtcCreateProgram")
    try:
        for e in expressions:
            ok(lib.nvrtcAddNameExpression(prog, f"&{e}".encode()), "nvrtcAddNameExpression")
        opts = (c_char_p * len(NVRTC_OPTIONS))(*[o.encode() for o in NVRTC_OPTIONS])
        rc = lib.nvrtcCompileProgram(prog, len(NVRTC_OPTIONS), opts)
        size = c_size_t()
        lib.nvrtcGetProgramLogSize(prog, ctypes.byref(size))
        buf = ctypes.create_string_buffer(size.value)
        lib.nvrtcGetProgramLog(prog, buf)
        log = buf.value.decode(errors="replace")
        if rc != 0:
            raise RuntimeError(f"NVRTC could not compile the objective:\n{log}\n--- source ---\n{source}")
        lowered = {}
        for e in expressions:
            name = c_char_p()
            ok(lib.nvrtcGetLoweredName(prog, f"&{e}".encode(), ctypes.byref(name)), "nvrtcGetLoweredName")
            lowered[e] = name.value.decode()
        ok(lib.nvrtcGetCUBINSize(prog, ctypes.byref(size)), "nvrtcGetCUBINSize")
        cubin = ctypes.create_string_buffer(size.value)
        ok(lib.nvrtcGetCUBIN(prog, cubin), "nvrtcGetCUBIN")
    finally:
        lib.nvrtcDestroyProgram(ctypes.byref(prog))
    return CompiledObjective(cubin.raw, [lowered[e] for e in expressions], _ptxas_info(log, lowered), time.perf_counter() - t0)


def register(cubin: bytes, names: list) -> int:
    """evok_objective_register: the id of the objective whose kernels (in EVOK_OBJ_KERNEL_* order) are in `cubin`."""
    arr = (c_char_p * len(names))(*[n.encode() for n in names])
    out = c_int()
    nat.check(nat.lib().evok_objective_register(cubin, len(cubin), arr, len(names), ctypes.byref(out)), "evok_objective_register")
    return out.value


def declare_data(objective_id: int, kinds: Dict[str, bool]) -> None:
    """evok_objective_declare_data: the registered id has these data names (True: a vector) and launches through instances only."""
    arr = (c_int * len(kinds))(*[int(v) for v in kinds.values()])
    nat.check(nat.lib().evok_objective_declare_data(objective_id, len(kinds), arr), "evok_objective_declare_data")


def bind_instance(base_id: int, ptrs: list, lens: list, item_strides: list, n_items: int) -> int:
    """evok_objective_instance: a new id with the kernels of `base_id` and this data binding (release it with `release_instance`)."""
    n = len(ptrs)
    out = c_int()
    rc = nat.lib().evok_objective_instance(base_id, (c_void_p * n)(*ptrs), (ctypes.c_int64 * n)(*lens), (ctypes.c_int64 * n)(*item_strides),
                                           n_items, n, ctypes.byref(out))
    nat.check(rc, "evok_objective_instance")
    return out.value


def release_instance(instance_id: int) -> None:
    nat.check(nat.lib().evok_objective_release(instance_id), "evok_objective_release")


def register_batched(objective_id: int, cubin: bytes, names: list) -> None:
    """evok_objective_register_batched: attach the batched kernels (in `batched_kernel_expressions` order) to a registered id."""
    arr = (c_char_p * len(names))(*[n.encode() for n in names])
    nat.check(nat.lib().evok_objective_register_batched(objective_id, cubin, len(cubin), arr, len(names)), "evok_objective_register_batched")


def register_eval_batched(objective_id: int, cubin: bytes, names: list) -> None:
    """evok_objective_register_eval_batched: attach the batched evaluation kernels (in `eval_batched_kernel_expressions` order)
    to a registered id."""
    arr = (c_char_p * len(names))(*[n.encode() for n in names])
    nat.check(nat.lib().evok_objective_register_eval_batched(objective_id, cubin, len(cubin), arr, len(names)),
              "evok_objective_register_eval_batched")


_cache: Dict[str, CompiledObjective] = {}
_batched_cache: Dict[str, CompiledObjective] = {}
_eval_batched_cache: Dict[str, CompiledObjective] = {}
_transform_cache: Dict[str, CompiledObjective] = {}
_cache_lock = threading.Lock()


def _declare(c: CompiledObjective, spec: ObjectiveSpec) -> None:
    if spec.kinds:
        declare_data(c.objective_id, spec.kinds)
    if spec.noisy:
        nat.check(nat.lib().evok_objective_declare_noise(c.objective_id), "evok_objective_declare_noise")


def compile_transform(spec: ObjectiveSpec) -> CompiledObjective:
    """Compile and register the objective of `spec` (one with a transform: `transform_kernel_expressions` are its kernels,
    evok_objective_register_transform), once per process for one generated source."""
    with _cache_lock:
        c = _transform_cache.get(spec.source)
        if c is None:
            c = compile_source(spec.source, transform_kernel_expressions())
            arr = (c_char_p * len(c.names))(*[n.encode() for n in c.names])
            out = c_int()
            nat.check(nat.lib().evok_objective_register_transform(c.cubin, len(c.cubin), arr, len(c.names), ctypes.byref(out)),
                      "evok_objective_register_transform")
            c.objective_id = out.value
            _declare(c, spec)
            _transform_cache[spec.source] = c
        return c


def compile_objective(spec: ObjectiveSpec) -> CompiledObjective:
    """Compile and register the objective of `spec`, once per process for one generated source."""
    with _cache_lock:
        c = _cache.get(spec.source)
        if c is None:
            c = compile_source(spec.source)
            c.objective_id = register(c.cubin, c.names)
            if spec.kinds:
                declare_data(c.objective_id, spec.kinds)
            if spec.noisy:
                nat.check(nat.lib().evok_objective_declare_noise(c.objective_id), "evok_objective_declare_noise")
            _cache[spec.source] = c
        return c


def compile_batched(spec: ObjectiveSpec) -> CompiledObjective:
    """Compile the batched samplers of `spec` and attach them to its registered id, once per process for one generated source."""
    base = compile_objective(spec)
    with _cache_lock:
        c = _batched_cache.get(spec.source)
        if c is None:
            c = compile_source(spec.source, batched_kernel_expressions())
            register_batched(base.objective_id, c.cubin, c.names)
            c.objective_id = base.objective_id
            _batched_cache[spec.source] = c
        return c


def compile_eval_batched(spec: ObjectiveSpec) -> CompiledObjective:
    """Compile the batched evaluation kernels of `spec` and attach them to its registered id, once per process for one generated
    source."""
    base = compile_objective(spec)
    with _cache_lock:
        c = _eval_batched_cache.get(spec.source)
        if c is None:
            c = compile_source(spec.source, eval_batched_kernel_expressions())
            register_eval_batched(base.objective_id, c.cubin, c.names)
            c.objective_id = base.objective_id
            _eval_batched_cache[spec.source] = c
        return c
