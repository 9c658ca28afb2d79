"""Host side of the descriptor regulariser in sparse mode (PointTexture.reg_loss -> train._RegLoss -> SparseRMSprop's dense-term
step): the gradient coefficient the backward records, restated in float32 and pinned to torch's CPU autograd of the reference's
expression bit for bit; the rule that picks the path; the C bindings."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from read_b200 import _lib, train
from read_b200.texture import PointTexture


def coef(u, w, numel):
    """k of the regulariser's gradient k * texture_ as torch's autograd forms it on the CPU for reg_weight * mean(texture_^2):
    MulBackward (u * fl32(w)), MeanBackward (/ fl32(numel)), PowBackward (2 * texture_, exact), all in float32."""
    uw = np.float32(u) * np.float32(w)
    return np.float32(2) * (uw / np.float32(numel))


def _autograd_grad(theta, w, u):
    p = theta.clone().requires_grad_(True)
    (w * p.square().mean()).backward(torch.tensor(u, dtype=torch.float32))
    return p.grad


@pytest.mark.parametrize("D, N", [(8, 5000), (1, 1_234_567), (1, 2 ** 24 + 1)])
@pytest.mark.parametrize("w, u", [(1e-3, 1.0), (1e-2, 0.37), (1.0, 1.0), (0.3, -2.5)])
def test_coefficient_restatement_equals_torch_cpu_autograd_bit_for_bit(D, N, w, u):
    theta = torch.rand((1, D, N), generator=torch.Generator().manual_seed(N % 1000)) * 4 - 2
    got = _autograd_grad(theta, w, u).numpy()
    k = coef(u, w, D * N)
    want = k * theta.numpy()                                       # fl(k * theta): float32 times float32 arrays
    assert want.dtype == np.float32
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    if float(np.float32(D * N)) != D * N:
        # numel not exact in float32: dividing by the exact numel instead gives other bits
        k_exact = np.float32(2) * np.float32(np.float64(np.float32(u) * np.float32(w)) / (D * N))
        assert k_exact != k and not np.array_equal(got, k_exact * theta.numpy())


def _tex(w=1e-2, n=64):
    return PointTexture(8, n, init_method='rand', reg_weight=w)


def test_reg_weight_zero_keeps_the_torch_expression():
    t = _tex(0.)
    train.request_sparse_grad(t)
    r = t.reg_loss()
    assert type(r.grad_fn).__name__ == "MulBackward0"
    assert float(r.detach()) == 0.0


def test_dense_optimizer_keeps_the_torch_expression():
    t = _tex()
    r = t.reg_loss()
    assert type(r.grad_fn).__name__ == "MulBackward0"
    assert torch.equal(r, 1e-2 * t.texture_.square().mean())


def test_no_grad_and_frozen_textures_keep_the_torch_expression():
    t = _tex()
    train.request_sparse_grad(t)
    with torch.no_grad():
        r = t.reg_loss()
    assert r.grad_fn is None and torch.equal(r, 1e-2 * t.texture_.square().mean())
    t.texture_.requires_grad_(False)
    assert t.reg_loss().grad_fn is None


def test_cpu_texture_in_sparse_mode_keeps_the_torch_expression():
    t = _tex()
    train.request_sparse_grad(t)                                   # NetAndTexture parks unloaded scenes on the CPU
    r = t.reg_loss()
    assert type(r.grad_fn).__name__ == "MulBackward0"
    r.backward()
    assert t.texture_.grad is not None and t.texture_.grad.shape == (1, 8, 64)


def test_null_grad_without_sparse_state():
    t = _tex()
    t.null_grad()
    assert t.texture_.grad is None


def test_bindings_are_declared():
    header = open(os.path.join(ROOT, "include", "read_b200.h")).read()
    for name in ("read_reg_loss_workspace_bytes", "read_reg_loss", "read_sparse_rmsprop_step_reg"):
        assert name in _lib.EXPORTS and f"{name}(" in header
    assert _lib._SIGS["read_reg_loss"][1][3] is __import__("ctypes").c_double
    assert len(_lib._SIGS["read_sparse_rmsprop_step_reg"][1]) == len(_lib._SIGS["read_sparse_rmsprop_step"][1]) + 1


def test_workspace_query_and_argument_checks():
    lib = _lib.load()
    assert lib.read_reg_loss_workspace_bytes(8, 5000) > 256
    assert lib.read_reg_loss_workspace_bytes(8, 5000) == lib.read_reg_loss_workspace_bytes(8, 2 ** 31 - 1)
    for D, N in [(0, 10), (17, 10), (8, 0)]:
        assert lib.read_reg_loss_workspace_bytes(D, N) == -1
    assert lib.read_reg_loss(None, 8, 10, 1.0, None, None, None) != 0                # rejected before any device work
    assert b"null" in lib.read_last_error()
    assert lib.read_sparse_rmsprop_step_reg(None, None, None, None, None, None, 10, 8, 1, 0.1, 0.99, 1e-8, 0.0, None, None) != 0
    assert b"null" in lib.read_last_error()
