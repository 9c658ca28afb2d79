"""Batches that mix scenes, host side (no GPU): the ctypes mirror of read_tex_table, and which batches NetAndTexture.forward runs as
one net call (the multi-texture gather) and which keep the per-item loop.  The gathers are replaced by CPU stand-ins and the net by
a counter, so only the dispatch is under test here; tests/test_gpu_multiscene.py checks the values on the GPU."""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn as nn

from conftest import ROOT
from read_b200 import _lib, compose, train as rtrain
from read_b200.compose import NetAndTexture
from read_b200.texture import PointTexture


def test_tex_table_mirror_matches_the_header_layout(tmp_path):
    fields = [n for n, _ in _lib.ReadTexTable._fields_]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "read_b200.h"', 'int main(void) {',
            '  printf("sizeof %zu\\n", sizeof(read_tex_table));',
            '  printf("slots %d\\n", READ_MAX_TEX_SLOTS);', '  printf("items %d\\n", READ_MAX_TEX_ITEMS);']
    prog += [f'  printf("{f} %zu\\n", offsetof(read_tex_table, {f}));' for f in fields]
    prog += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["sizeof"]) == ctypes.sizeof(_lib.ReadTexTable)
    assert (int(got["slots"]), int(got["items"])) == (_lib.MAX_TEX_SLOTS, _lib.MAX_TEX_ITEMS)
    for f in fields:
        assert int(got[f]) == getattr(_lib.ReadTexTable, f).offset, f


class CountingNet(nn.Module):
    """Stands in for the UNet: counts calls and returns zeros of the RGB shape."""

    def __init__(self, train_batchnorm='batch'):
        super().__init__()
        self.calls, self.train_batchnorm = [], train_batchnorm

    def forward(self, *xs, **kwargs):
        self.calls.append(xs[0].shape[0])
        return torch.zeros((xs[0].shape[0], 3) + tuple(xs[0].shape[2:]))


@pytest.fixture
def cpu_gathers(monkeypatch):
    """CPU stand-ins for the gathers; each records the batch size it sampled."""
    seen = []

    def one(self, inputs):
        seen.append(('one', inputs.shape[0]))
        return torch.zeros((inputs.shape[0], self.texture_.shape[1]) + tuple(inputs.shape[2:]))

    def items(textures, slots, inputs):
        seen.append(('items', inputs.shape[0]))
        return torch.zeros((inputs.shape[0], 8) + tuple(inputs.shape[2:]))

    monkeypatch.setattr(PointTexture, "forward", one)
    monkeypatch.setattr(compose, "sample_items", items)
    return seen


def _model(n_tex=3, net=None, **kw):
    texs = {i: PointTexture(8, 50 + i, **kw) for i in range(n_tex)}
    m = NetAndTexture(net or CountingNet(), texs)
    m.load_textures(list(texs))
    return m


def _inputs(ids, S=32):
    B = len(ids)
    return {'uv_1d_p1': torch.zeros((B, 1, S, S)), 'uv_1d_p1_ds1': torch.zeros((B, 1, S // 2, S // 2)), 'id': torch.tensor(ids)}


def test_table_maps_items_to_slots_in_first_appearance_order():
    m = _model()
    textures, slots = m._texture_table([0, 1, 0, 2, 1])
    assert textures == [m._texture(0), m._texture(1), m._texture(2)]
    assert slots == [0, 1, 0, 2, 1]
    textures, slots = m._texture_table([2, 2, 0])
    assert textures == [m._texture(2), m._texture(0)] and slots == [0, 0, 1]
    assert m._texture_table([1, 1]) is None                         # one texture: its own path


def test_table_refuses_what_the_kernels_do_not_take():
    m = _model()
    m._texture(1).activation = 'sigmoid'
    assert m._texture_table([0, 1]) is None                          # differing activation
    assert m._texture_table([0, 2]) is not None
    m = _model()
    rtrain.request_sparse_grad(m._texture(0))
    assert m._texture_table([0, 1]) is None                          # sparse and dense
    rtrain.request_sparse_grad(m._texture(1))
    assert m._texture_table([0, 1]) is not None
    m = _model()
    m._texture(2).texture_.requires_grad_(False)
    assert m._texture_table([0, 2]) is None                          # one texture needs a gradient, the other not
    m = _model(n_tex=17)
    assert m._texture_table(list(range(17))) is None                 # more than 16 textures
    assert m._texture_table(list(range(16))) is not None
    assert m._texture_table([0, 1] * 33) is None                     # more than 64 items
    assert m._texture_table([0, 1] * 32) is not None
    m = NetAndTexture(CountingNet(), {0: PointTexture(8, 10), 1: PointTexture(4, 10)})
    m.load_textures([0, 1])
    assert m._texture_table([0, 1]) is None                          # D != 8


@pytest.mark.parametrize("mode", ["eval", "train per_item"])
def test_mixed_batch_is_one_net_call(cpu_gathers, mode):
    net = CountingNet('per_item' if mode != "eval" else 'batch')
    m = _model(net=net)
    m.train(mode != "eval")
    out, net_input = m(_inputs([0, 1, 0, 2, 1]), return_input=True)
    assert net.calls == [5] and tuple(out.shape) == (5, 3, 32, 32)
    assert cpu_gathers == [('items', 5), ('items', 5)]               # one gather per 'uv' key
    assert [tuple(t.shape) for t in net_input] == [(1, 8, 32, 32), (1, 8, 16, 16)]   # the last item's input


def test_one_texture_keeps_its_path(cpu_gathers):
    net = CountingNet()
    m = _model(net=net).eval()
    m(_inputs([1, 1, 1]))
    assert net.calls == [3] and cpu_gathers == [('one', 3), ('one', 3)]


def _loop_calls(m, ids, seen):
    net = m.net
    net.calls.clear()
    seen.clear()
    m(_inputs(ids))
    return net.calls, {k for k, _ in seen}


def test_fallbacks_take_the_loop(cpu_gathers):
    ids = [0, 1, 0, 2]
    loop = ([1, 1, 1, 1], {'one'})
    m = _model().eval()
    m.temporal_average = True
    assert _loop_calls(m, ids, cpu_gathers) == loop                  # temporal average
    m = _model().train()                                             # train() with call-wide BatchNorm statistics
    assert _loop_calls(m, ids, cpu_gathers) == loop
    m = _model().eval()
    m._texture(2).activation = 'tanh'
    assert _loop_calls(m, ids, cpu_gathers) == loop                  # differing activation
    m = _model(n_tex=17).eval()
    assert _loop_calls(m, list(range(17)), cpu_gathers) == ([1] * 17, {'one'})     # more than 16 textures
    m = _model().eval()
    rtrain.request_sparse_grad(m._texture(0))
    assert _loop_calls(m, ids, cpu_gathers) == loop                  # sparse and dense
    m = _model().eval()
    assert _loop_calls(m, ids, cpu_gathers) == ([4], {'items'})      # and the same model without any of them: one call
