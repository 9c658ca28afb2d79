"""Descriptor side of the training step on our kernels (SURVEY.md §8f rank 2, §8e "Training").

The reference trains the per-point descriptors with autograd through ``PointTexture.forward`` (a dense ``[D, B*N]`` ``index_add_``
per pyramid level, READ/models/texture.py:55-63) and a dense ``torch.optim.RMSprop`` over all N points (READ/pipelines/ogl.py:16,
97-102,129-144; the step itself is src/train.py:257-266).  Only the few 10^4 points visible in the batch receive a gradient, so:

* ``enable_sparse_grad(texture)`` switches a ``PointTexture`` to a backward that scatter-adds into a persistent point-major
  accumulator and flags the touched points (``texture_.grad`` stays ``None``: nothing dense is ever materialised);
* ``SparseRMSprop`` is a drop-in for the reference's descriptor optimizer (same hyper-parameters, ``param_groups`` whose ``lr`` the
  pipeline rescales, ``step() / zero_grad() / state_dict()``): it updates only touched points, with the skipped ``square_avg``
  decays applied lazily - the result equals the dense optimizer's.  With weight decay every point has a gradient, so every
  point is updated on every step.  ``PointTexture.reg_loss`` (``--reg_weight``) in sparse mode
  back-propagates one scalar per texture (``_RegLoss``), and the step after it updates every point with that term added;
* ``exchange_sparse_grads`` is the data-parallel join: ranks all-gather their touched ``(id, grad[D])`` rows (a few MB) instead
  of all-reducing ``[N, D]`` gradients or re-broadcasting the texture as ``nn.DataParallel`` does (train.py:138-139).

The net's own backward still runs through torch's operators (library path, DESIGN.md §7).
"""
import ctypes
import warnings

import torch
from torch.autograd.function import once_differentiable

from . import _lib as L
from . import ops


class _GatherSparse(torch.autograd.Function):
    """PointTexture sampling whose backward accumulates into the texture's sparse-gradient state."""

    @staticmethod
    def forward(ctx, texture_, ids, tex_module):
        ctx.save_for_backward(ids)
        ctx.tex = tex_module
        return ops.gather_from_index(tex_module.point_major(), ids, L.FEAT_NCHW_F32)

    @staticmethod
    def backward(ctx, grad_out):
        (ids,) = ctx.saved_tensors
        st = ctx.tex._sparse
        g = grad_out.contiguous()
        if g.dtype != torch.float32:
            g = g.float()
        ops.gather_backward_sparse(g, ids, st.N, st.grad, st.touched)
        return None, None, None


class _RegLoss(torch.autograd.Function):
    """``PointTexture.reg_loss`` (reg_weight * mean(texture_^2), READ/models/texture.py:40-41) in sparse mode.  Its gradient is
    k * texture_ with k = 2 * u * reg_weight / numel for the upstream gradient u, so the backward records the scalar k in the
    texture's sparse state (summed over calls) instead of a dense [1, D, N] gradient; SparseRMSprop.step applies it to every point.
    k is computed with the device ops autograd runs for the torch expression (u * w, / numel, * 2), so k * texture_ has the bits of
    the gradient autograd would give."""

    @staticmethod
    def forward(ctx, texture_, tex_module):
        p = texture_.detach()
        D, N = p.shape[1], p.shape[2]
        ctx.tex, ctx.w, ctx.numel = tex_module, float(tex_module.reg_weight), D * N
        lib = L.load()
        ws = torch.empty(int(lib.read_reg_loss_workspace_bytes(D, N)), dtype=torch.uint8, device=p.device)
        out = torch.empty((), dtype=torch.float32, device=p.device)
        L.check(lib.read_reg_loss(p.data_ptr(), D, N, ctx.w, out.data_ptr(), ws.data_ptr(), L.stream_ptr()))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, u):
        sp = enable_sparse_grad(ctx.tex)
        k = u * ctx.w / ctx.numel * 2
        sp.reg_coef = k if sp.reg_coef is None else sp.reg_coef + k
        return None, None


class SparseGradState:
    def __init__(self, texture):
        p = texture.texture_
        if not p.is_cuda:
            raise RuntimeError("read_b200.train: the texture must be on a CUDA device (no CPU fallback)")
        self.D, self.N = p.shape[1], p.shape[2]
        self.grad = torch.zeros((self.N, self.D), dtype=torch.float32, device=p.device)       # point-major accumulator
        self.touched = torch.zeros((self.N,), dtype=torch.uint8, device=p.device)
        self.reg_coef = None        # 0-d device f32: the pending regulariser's gradient coefficient k (_RegLoss), or None


def enable_sparse_grad(texture):
    """Route ``texture``'s backward into a sparse accumulator (idempotent); returns the state.  The buffers live on the texture's
    CUDA device; for textures still parked on the CPU (NetAndTexture keeps unloaded scenes there) use ``request_sparse_grad``."""
    texture._sparse_requested = True
    st = getattr(texture, "_sparse", None)
    if st is None or st.grad.device != texture.texture_.device:
        st = texture._sparse = SparseGradState(texture)
    return st


def request_sparse_grad(texture):
    """Mark ``texture`` for sparse gradients; the state is created on its first CUDA forward."""
    texture._sparse_requested = True


def disable_sparse_grad(texture):
    texture._sparse = None
    texture._sparse_requested = False


def touched_count(texture):
    return int(texture._sparse.touched.sum().item())


class SparseRMSprop:
    """RMSprop (torch defaults: alpha 0.99, eps 1e-8, no momentum, not centered) over PointTexture descriptors, touching only the
    points that received a gradient since the last step.  ``textures``: one PointTexture or a list (one param group each, like the
    reference's multi-scene ``extra_optimizer``, ogl.py:136-144).  A texture whose regulariser was back-propagated since its last
    step (a pending ``reg_coef``) gets the dense-term step instead: every point, with g = accumulated row + reg_coef * param.
    A param group with ``weight_decay != 0`` takes that every-point step on every step (with a zero coefficient when no
    regulariser is pending): torch.optim.RMSprop adds weight_decay * param to the zero gradient of a point outside the batch, so
    with weight decay every point moves every step, and skipping the untouched ones would not give the dense optimizer's result."""

    def __init__(self, textures, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0.0):
        if not isinstance(textures, (list, tuple)):
            textures = [textures]
        self.textures = list(textures)
        self.defaults = dict(lr=lr, alpha=alpha, eps=eps, weight_decay=weight_decay)
        self.param_groups = [dict(self.defaults, params=[t.texture_]) for t in self.textures]
        self.state = {}
        self._steps = 0
        for t in self.textures:
            request_sparse_grad(t)

    def _state(self, t):
        st = self.state.get(id(t))
        if st is None or st["square_avg"].device != t.texture_.device:
            sp = t._sparse
            st = self.state[id(t)] = {"square_avg": torch.zeros((sp.N, sp.D), dtype=torch.float32, device=t.texture_.device),
                                      "last_step": torch.zeros((sp.N,), dtype=torch.int32, device=t.texture_.device)}
        return st

    def _zero_coef(self, t):
        z = getattr(self, "_zero", None)
        if z is None or z.device != t.texture_.device:
            z = self._zero = torch.zeros((), dtype=torch.float32, device=t.texture_.device)
        return z

    def zero_grad(self, set_to_none=True):
        """Gradient rows are cleared by ``step`` itself; calling this before the first backward is harmless."""
        for t in self.textures:
            t.texture_.grad = None

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self._steps += 1
        lib, sp_ = L.load(), L.stream_ptr()
        for t, g in zip(self.textures, self.param_groups):
            sp, st = enable_sparse_grad(t), self._state(t)
            shadow = t.point_major()                 # kept in sync by the kernel: no dense re-transposition after the step
            args = (t.texture_.data_ptr(), shadow.data_ptr(), sp.grad.data_ptr(), sp.touched.data_ptr(), st["square_avg"].data_ptr(),
                    st["last_step"].data_ptr(), sp.N, sp.D, self._steps, float(g["lr"]), float(g["alpha"]), float(g["eps"]),
                    float(g["weight_decay"]))
            if sp.reg_coef is not None:              # the regulariser's gradient reaches every point: the dense-term step
                coef, sp.reg_coef = sp.reg_coef, None
                L.check(lib.read_sparse_rmsprop_step_reg(*args, coef.data_ptr(), sp_))
            elif float(g["weight_decay"]) != 0.0:    # so does weight decay's: the same step with a zero coefficient
                L.check(lib.read_sparse_rmsprop_step_reg(*args, self._zero_coef(t).data_ptr(), sp_))
            else:
                L.check(lib.read_sparse_rmsprop_step(*args, sp_))
        return loss

    def dense_square_avg(self, t):
        """[1,D,N] square_avg exactly as the dense torch.optim.RMSprop would hold it now (lazy decays applied)."""
        sp, st = t._sparse, self._state(t)
        out = torch.empty((1, sp.D, sp.N), dtype=torch.float32, device=t.texture_.device)
        L.check(L.load().read_square_avg_dense(st["square_avg"].data_ptr(), st["last_step"].data_ptr(), sp.N, sp.D, self._steps,
                                               float(self.defaults["alpha"]), out.data_ptr(), L.stream_ptr()))
        return out

    def state_dict(self):
        """torch.optim.RMSprop's layout ({'state': {i: {'step', 'square_avg'}}, 'param_groups': ...}) so that checkpoints written
        by train.py stay loadable by either optimizer."""
        state = {i: {"step": torch.tensor(float(self._steps)), "square_avg": self.dense_square_avg(t).cpu()}
                 for i, t in enumerate(self.textures)}
        groups = [{k: v for k, v in g.items() if k != "params"} | {"params": [i]} for i, g in enumerate(self.param_groups)]
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        for i, t in enumerate(self.textures):
            s = sd["state"].get(i)
            if s is None:
                continue
            st = self._state(t)
            self._steps = int(s["step"])
            sq = s["square_avg"].to(t.texture_.device, torch.float32).reshape(t._sparse.D, t._sparse.N)
            st["square_avg"].copy_(sq.t())
            st["last_step"].fill_(self._steps)
        for g, gs in zip(self.param_groups, sd.get("param_groups", [])):
            g.update({k: v for k, v in gs.items() if k != "params"})


def exchange_sparse_grads(texture, group=None, capacity=None):
    """Data-parallel join of the descriptor gradients: every rank contributes its touched (id, grad[D]) rows, every rank ends up
    with the SUM over ranks in its accumulator (and the union of the flags) - what all-reducing the dense [N,D] gradient would
    give, for a few MB of traffic.  Returns the number of rows this rank sent.

    The compaction and the scatter of received rows use atomics, so the accumulator's last bits can vary from run to run.  Under
    torch.use_deterministic_algorithms(True) this raises a RuntimeError before any communication, as torch does for its own
    nondeterministic ops; with warn_only=True it warns instead and proceeds."""
    if torch.are_deterministic_algorithms_enabled():
        msg = ("read_b200.train.exchange_sparse_grads does not have a deterministic implementation, but you set "
               "'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you can use "
               "the 'warn_only=True' option, if that's acceptable for your application.")
        if not torch.is_deterministic_algorithms_warn_only_enabled():
            raise RuntimeError(msg)
        warnings.warn(msg)
    import torch.distributed as dist
    sp = enable_sparse_grad(texture)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return touched_count(texture)
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lib, dev = L.load(), sp.grad.device
    cap = int(capacity) if capacity else max(1024, touched_count(texture))
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    ids = torch.empty(cap, dtype=torch.int32, device=dev)
    grads = torch.empty((cap, sp.D), dtype=torch.float32, device=dev)
    L.check(lib.read_compact_touched(sp.grad.data_ptr(), sp.touched.data_ptr(), sp.N, sp.D, cnt.data_ptr(), cap, ids.data_ptr(),
                                     grads.data_ptr(), L.stream_ptr()))
    n_mine = min(int(cnt.item()), cap)
    counts = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(world)]
    dist.all_gather(counts, torch.tensor([n_mine], dtype=torch.int32, device=dev), group=group)
    n_max = max(int(c.item()) for c in counts)
    if n_max == 0:
        return 0
    if cap < n_max:                                   # pad to the common length of the all-gather
        ids = torch.cat([ids[:n_mine], torch.zeros(n_max - n_mine, dtype=torch.int32, device=dev)])
        grads = torch.cat([grads[:n_mine], torch.zeros((n_max - n_mine, sp.D), dtype=torch.float32, device=dev)])
    all_ids = torch.empty((world, n_max), dtype=torch.int32, device=dev)
    all_grads = torch.empty((world, n_max, sp.D), dtype=torch.float32, device=dev)
    if dist.get_backend(group) == "gloo":
        li, lg = [torch.empty_like(all_ids[0]) for _ in range(world)], [torch.empty_like(all_grads[0]) for _ in range(world)]
        dist.all_gather(li, ids[:n_max].contiguous(), group=group)
        dist.all_gather(lg, grads[:n_max].contiguous(), group=group)
        all_ids, all_grads = torch.stack(li), torch.stack(lg)
    else:
        dist.all_gather_into_tensor(all_ids, ids[:n_max].contiguous(), group=group)
        dist.all_gather_into_tensor(all_grads, grads[:n_max].contiguous(), group=group)
    for r in range(world):
        n_r = int(counts[r].item())
        if r == rank or n_r == 0:
            continue
        L.check(lib.read_scatter_pairs(all_ids[r].data_ptr(), all_grads[r].data_ptr(), n_r, sp.D, sp.N, sp.grad.data_ptr(),
                                       sp.touched.data_ptr(), L.stream_ptr()))
    return n_mine
