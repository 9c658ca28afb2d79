"""Drop-in for ``READ.gl.myrender.MyRender`` (src/READ/gl/myrender.py:12-43), on the H100 kernels.

Differences in HOW (not WHAT): the point clouds are uploaded once in ``update_ds`` and stay resident in HBM
(the reference re-uploads N*12 bytes per level per call, pcpr_cuda.cpp:29); all L levels and all views of a
dataset id are produced by ONE pass over the points (the reference projects every point L times); outputs are
bit-identical to a sequential execution of the reference kernel.
"""
import numpy as np
import torch

from . import ops
from . import _lib as L

inv = np.linalg.inv


class MyRender:
    def __init__(self, ds_list=None, device_outputs=False):
        self.device_outputs = device_outputs
        self._pyr = {}
        if ds_list:
            self.update_ds(ds_list)

    def update_ds(self, ds_list):
        L.require_device()
        self.ds_list = ds_list
        self.ds_ids = [d.id for d in ds_list]
        self.tgt_sh = self.ds_list[0].tgt_sh
        dev = torch.device("cuda", torch.cuda.current_device())
        self.points = {
            ds.id: torch.from_numpy(np.ascontiguousarray(np.asarray(ds.scene_data['pointcloud']['xyz']), dtype=np.float32)).to(dev)
            for ds in ds_list}

    def _pyramid(self, B, W, H, n_levels, dev):
        key = (B, W, H, n_levels, dev)
        if key not in self._pyr:
            self._pyr[key] = ops.Pyramid(B, W, H, n_levels, dev)
        return self._pyr[key]

    def render(self, data):
        input_format = self.ds_list[0].input_format.replace(' ', '').split(',')
        n_levels = len(input_format)
        ids = data['input']['id']
        ids_t = torch.as_tensor(ids).reshape(-1)
        nb = ids_t.shape[0]
        out_dict, depth_dict = {'id': ids}, {}

        proj_matrix = np.asarray(data['proj_matrix'], dtype=np.float32).reshape(-1, 4, 4)
        view_matrix = np.asarray(data['view_matrix'], dtype=np.float32).reshape(-1, 4, 4)
        total_m = torch.from_numpy(proj_matrix @ inv(view_matrix))          # myrender.py:28-30, same numpy call

        W, H = int(self.tgt_sh[0]), int(self.tgt_sh[1])
        sizes = ops.level_sizes(W, H, n_levels)
        dev = next(iter(self.points.values())).device
        idx_levels = [torch.zeros((nb, h, w), dtype=torch.float32, device=dev) for (w, h) in sizes]
        dep_levels = [torch.zeros((nb, h, w), dtype=torch.float32, device=dev) for (w, h) in sizes]
        for ds_id in self.ds_ids:
            sel = torch.where(ids_t == ds_id)[0]
            if sel.numel() == 0:
                continue
            m = total_m[sel].contiguous().to(dev)
            pyr = self._pyramid(int(sel.numel()), W, H, n_levels, dev)
            pyr.clear()
            ops.raster_project(pyr, self.points[ds_id], m)
            sel_d = sel.to(dev)
            for l in range(n_levels):
                i, d = ops.zbuf_resolve(pyr, l)
                idx_levels[l][sel_d] = i
                dep_levels[l][sel_d] = d
        for l, k in enumerate(input_format):
            i, d = idx_levels[l].unsqueeze(1), dep_levels[l].unsqueeze(1)
            if not self.device_outputs:
                i, d = i.cpu(), d.cpu()
            out_dict[k] = i
            depth_dict[k] = d
        return out_dict, depth_dict
