"""Batched flat-parameter policies (mirrors `Policy` of evotorch.neuroevolution.net.vecrl, vecrl.py:1019-1300, and the
helpers of net/misc.py).

A `Policy` wraps a torch module; `set_parameters(P)` takes either one flat parameter vector (length L) or an N x L matrix
(one row per solution of the population), and `policy(obs)` then applies row i of P to row i of `obs`.  The reference does
this with `vmap(functional_call)` (vecrl.py:1264).  Here, feed-forward nets made of `Linear` layers and Tanh / ReLU /
Sigmoid / Identity activations run on the K8 kernel (csrc/evok_mlp.cu) for CUDA float32 tensors: every parameter row is read
from HBM exactly once.  Any other stateless module (custom layers) or device takes the generic torch.func path; stateful
(recurrent) modules are rejected, because the per-environment hidden-state handling of the reference is not implemented.
"""

from __future__ import annotations

from typing import Optional

import torch
from torch import nn
from torch.func import functional_call, vmap

from .. import ops

_ACTS = {nn.Tanh: "tanh", nn.ReLU: "relu", nn.Sigmoid: "sigmoid", nn.Identity: "none"}


def count_parameters(net: nn.Module) -> int:
    """Total number of (trainable or not) parameters (net/misc.py `count_parameters`)."""
    return sum(p.numel() for p in net.parameters())


@torch.no_grad()
def parameter_vector(net: nn.Module) -> torch.Tensor:
    """All parameters flattened in `parameters()` order (net/misc.py `parameter_vector`)."""
    return torch.cat([p.reshape(-1) for p in net.parameters()])


@torch.no_grad()
def fill_parameters(net: nn.Module, vector: torch.Tensor):
    """Write a flat vector into the module's parameters (net/misc.py `fill_parameters`)."""
    offset = 0
    for p in net.parameters():
        n = p.numel()
        p.copy_(vector[offset:offset + n].reshape(p.shape))
        offset += n
    if offset != vector.numel():
        raise ValueError(f"The parameter vector has {vector.numel()} elements, the network needs {offset}.")


def _feedforward_spec(net: nn.Module) -> Optional[tuple]:
    """(layer widths, activations) if `net` is a Sequential of Linear(+bias) layers with supported activations, else None."""
    from .net.multilayered import MultiLayered  # what str_to_net("A >> B >> C") builds

    if isinstance(net, nn.Linear):
        layers = [net]
    elif isinstance(net, (nn.Sequential, MultiLayered)):
        layers = list(net)
    else:
        return None
    dims, acts = [], []
    for m in layers:
        if isinstance(m, nn.Linear):
            if m.bias is None:
                return None
            if dims and dims[-1] != m.in_features:
                return None
            if not dims:
                dims.append(m.in_features)
            dims.append(m.out_features)
            acts.append("none")
        elif type(m) in _ACTS:
            if not acts or acts[-1] != "none":
                if type(m) is nn.Identity:
                    continue
                return None
            acts[-1] = _ACTS[type(m)]
        else:
            return None
    if not acts or len(acts) > 8 or max(dims) > 2048:
        return None
    return dims, acts


class Policy:
    """A (batch of) policies sharing one network architecture, parameterised by flat vectors (vecrl.py:1019)."""

    def __init__(self, net: nn.Module):
        for m in net.modules():
            if isinstance(m, (nn.RNNBase, nn.RNNCellBase)):
                # the reference's Policy carries hidden states across calls and resets them per environment (vecrl.py:1160-1238);
                # that state handling is not implemented here, and silently running a recurrent net without it would be wrong
                raise NotImplementedError(f"Policy does not support stateful (recurrent) modules: found {type(m).__name__}")
        self._net = net
        self._names = [name for name, _ in net.named_parameters()]
        self._shapes = [p.shape for _, p in net.named_parameters()]
        self._sizes = [p.numel() for _, p in net.named_parameters()]
        self._spec = _feedforward_spec(net)
        self._parameters: Optional[torch.Tensor] = None

    @property
    def parameter_length(self) -> int:
        return sum(self._sizes)

    @property
    def parameters(self) -> Optional[torch.Tensor]:
        return self._parameters

    def set_parameters(self, parameters: torch.Tensor, indices=None, *, reset: bool = True):
        """One flat vector (shared by every observation) or an N x L matrix (row i drives observation i) (vecrl.py:1138)."""
        if parameters.shape[-1] != self.parameter_length or parameters.ndim not in (1, 2):
            raise ValueError(f"Expected parameters of shape (L,) or (N, L) with L = {self.parameter_length}, got {tuple(parameters.shape)}")
        if indices is not None:
            self._parameters[torch.as_tensor(indices)] = parameters
        else:
            self._parameters = parameters

    def _unflatten(self, flat: torch.Tensor) -> dict:
        out, offset = {}, 0
        for name, shape, size in zip(self._names, self._shapes, self._sizes):
            out[name] = flat[offset:offset + size].reshape(shape)
            offset += size
        return out

    def _call_one(self, flat: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
        return functional_call(self._net, self._unflatten(flat), (x,))

    @torch.no_grad()
    def forward_shared(self, parameters: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
        """Row i of `parameters` (N x L) applied to the SAME input batch `x` (B x in) -> N x B x out: a population scored on a
        common minibatch (supervisedne.py:337-347).  For feed-forward nets on CUDA float32 the layers run on the kernels of
        `ops.mlp_forward_shared` (first layer: one tensor-core product of the stacked weight rows of all N networks with the
        shared batch); anything else, including nets those kernels cannot take (`ops.mlp_forward_shared_supported`), goes
        through `vmap(functional_call)`."""
        if parameters.ndim != 2 or parameters.shape[1] != self.parameter_length:
            raise ValueError(f"Expected parameters of shape (N, {self.parameter_length}), got {tuple(parameters.shape)}")
        if self._spec is not None and ops.uses_kernels(parameters) and ops.uses_kernels(x) and x.ndim == 2 and parameters.stride(1) == 1:
            dims, acts = self._spec
            if ops.mlp_forward_shared_supported(dims):
                return ops.mlp_forward_shared(parameters, x.contiguous(), dims, acts)
        return vmap(self._call_one, in_dims=(0, None))(parameters, x)

    @torch.no_grad()
    def __call__(self, x: torch.Tensor, *, obs_norm=None, active: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Row i of the parameters applied to observation i (vecrl.py:1240-1279).  Rollout extras, fused into the K8 kernel
        on CUDA float32: `obs_norm` (a RunningNorm) normalises and clips the observations on the fly, `active` (bool, N)
        skips the policies of finished sub-environments (zero actions; their parameters are not read)."""
        p = self._parameters
        if p is None:
            raise ValueError("Please use the method `set_parameters(...)` before calling the policy.")
        if p.ndim == 1:
            if obs_norm is not None:
                x = obs_norm.normalize(x)
            return self._call_one(p, x)
        if x.ndim != 2 or x.shape[0] != p.shape[0]:
            raise ValueError(f"With {p.shape[0]} parameter rows, expected observations of shape ({p.shape[0]}, ...), got {tuple(x.shape)}")
        if self._spec is not None and ops.uses_kernels(p) and ops.uses_kernels(x) and p.stride(1) == 1 and x.stride(1) == 1:
            dims, acts = self._spec
            if obs_norm is None:
                return ops.mlp_forward(p, x, dims, acts, active=active)
            if obs_norm.sum is None:
                raise ValueError("Cannot do normalization because no data is collected yet.")
            return ops.mlp_forward(p, x, dims, acts, obs_sum=obs_norm.sum, obs_sumsq=obs_norm.sum_of_squares, obs_count=obs_norm.count_tensor,
                                   min_variance=obs_norm.min_variance, clip=(obs_norm.low, obs_norm.high), active=active)
        if obs_norm is not None:
            x = obs_norm.normalize(x)
        result = vmap(self._call_one)(p, x)
        if active is not None:
            result = torch.where(active.reshape((-1,) + (1,) * (result.ndim - 1)), result, torch.zeros_like(result))
        return result
