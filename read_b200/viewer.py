"""Viewer-side renderer: the device-resident replacement for ``READ.gl.nn.OGL`` (READ/gl/nn.py:76-129).

The reference's ``OGL`` draws index maps with OpenGL (``MultiscaleRender``), runs ``model(input_dict, return_input=True)``
and returns ``{'output': [H,W,4] f32 on the GPU (RGB + alpha 1), 'net_input': ...}`` (nn.py:113-129); ``viewer.py:267``
then flips the frame vertically for display.  ``FrameRenderer`` keeps that output contract but needs no OpenGL: one
pass over the point cloud on the GPU (``NetAndTexture.render``) and ONE small kernel that writes the displayable
``[H,W,4]`` surface (alpha, optional vertical flip) straight from the net's output planes.
"""
import numpy as np
import torch

from . import _lib as L
from . import ops
from .compose import NetAndTexture
from .texture import PointTexture
from .unet import UNet


class FrameRenderer:
    def __init__(self, xyz, net_state_dict, texture, viewport_size, supersampling=1, temporal_average=False,
                 device=None, flip_vertical=False, n_levels=4, return_net_input=True):
        """xyz: [N,3] float32 (numpy / tensor); net_state_dict: UNet checkpoint ``state_dict``; texture: the
        ``[1,8,N]`` descriptor tensor (``PointTexture.texture_``) or a ``PointTexture``; viewport_size: (W, H) of the output
        frame.  ``supersampling`` / ``temporal_average``: the options of READ/gl/nn.py:76,100-103 (the pyramid is rendered at
        ss x the viewport and reduced bilinearly; every level is averaged with the previous frame's input), served on the fused
        path.  ``return_net_input=False`` skips materialising the reference's ``net_input`` list (4 small transposes)."""
        W, H = int(viewport_size[0]), int(viewport_size[1])
        factor = 16
        assert W % 16 == 0, f'set width {factor * (W // factor)}'          # READ/gl/nn.py:107-109
        assert H % 16 == 0, f'set height {factor * (H // factor)}'
        assert int(supersampling) >= 1, 'supersampling must be a positive integer'
        L.require_device(None if device is None else torch.device(device).index)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.W, self.H, self.n_levels = W, H, n_levels
        self.flip_vertical = bool(flip_vertical)
        xyz = torch.as_tensor(np.asarray(xyz, dtype=np.float32) if not torch.is_tensor(xyz) else xyz, dtype=torch.float32)
        self.xyz = xyz.contiguous().to(self.device)
        # scene load: spatially sorted device store (original ids travel with the points), see ops.SortedPoints
        ss = int(supersampling)
        nested = L.load().read_raster_direct_mask(W * ss, H * ss, n_levels) == 1   # every level exactly half of the previous one
        self.store = ops.SortedPoints(self.xyz) if nested else None
        net = UNet()
        net.load_state_dict(net_state_dict, strict=True)
        if not isinstance(texture, PointTexture):
            t = torch.as_tensor(texture, dtype=torch.float32)
            assert t.dim() == 3 and t.shape[0] == 1 and t.shape[2] == self.xyz.shape[0], "texture must be [1,D,N]"
            tex = PointTexture(t.shape[1], t.shape[2])
            with torch.no_grad():
                tex.texture_.copy_(t)
            texture = tex
        self.model = NetAndTexture(net, {0: texture}, ss, temporal_average=bool(temporal_average))
        self.return_net_input = bool(return_net_input)
        self.model.load_textures(0)
        self.model.to(self.device).eval()
        # camera upload: a ring of pinned 4x4 staging buffers.  A pageable ``.to(device)`` blocks the host until the copy has run,
        # and the copy is queued behind the previous frame's kernels - the host could not enqueue frame i+1 while frame i renders
        # and the GPU idled for the host-side work of every frame.
        self._cam_host = [torch.empty((1, 4, 4), dtype=torch.float32).pin_memory() for _ in range(4)]
        self._cam_used = [None] * 4
        self._cam_i = 0

    def _upload_camera(self, total_m):
        i = self._cam_i
        self._cam_i = (i + 1) % len(self._cam_host)
        if self._cam_used[i] is not None:
            self._cam_used[i].synchronize()              # the copy that last read this staging buffer (4 frames ago) has run
        self._cam_host[i].copy_(torch.from_numpy(total_m.reshape(1, 4, 4)))
        m = self._cam_host[i].to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._cam_used[i] = ev
        return m

    @classmethod
    def from_checkpoints(cls, xyz, net_ckpt, texture_ckpt, viewport_size, **kw):
        """The reference's checkpoint format: ``{'state_dict': ..., 'args': ...}`` (READ/utils/train.py:42-65)."""
        net_sd = torch.load(net_ckpt, map_location="cpu")["state_dict"]
        tex_sd = torch.load(texture_ckpt, map_location="cpu")["state_dict"]
        return cls(xyz, net_sd, tex_sd["texture_"], viewport_size, **kw)

    @staticmethod
    def total_matrix(proj_matrix, view_matrix):
        """proj @ inv(view) in float32 on the host, the call src/READ/gl/myrender.py:28-30 makes."""
        proj = np.asarray(proj_matrix, dtype=np.float32)
        view = np.asarray(view_matrix, dtype=np.float32)
        return (proj @ np.linalg.inv(view)).astype(np.float32)

    def infer(self, proj_matrix, view_matrix):
        """-> {'output': [H,W,4] f32 cuda tensor (RGB, alpha 1; flipped if ``flip_vertical``), 'net_input': list of the four
        [1,8,h,w] f32 net inputs (None with ``return_net_input=False``)} - the contract of ``OGL.infer`` (READ/gl/nn.py:113-129).
        Both are fresh tensors: the caller may keep them across frames, as with the reference."""
        m = self._upload_camera(self.total_matrix(proj_matrix, view_matrix))
        with torch.no_grad():
            res = self.model.render(self.store if self.store is not None else self.xyz, m, self.W, self.H,
                                    n_levels=self.n_levels, return_input=self.return_net_input, clone_output=False)
        out, net_input = res if self.return_net_input else (res, None)                       # out: [1,3,H,W] f32
        rgba = torch.empty((self.H, self.W, 4), dtype=torch.float32, device=self.device)
        L.check(L.load().read_frame_to_rgba(out.data_ptr(), self.H, self.W, int(self.flip_vertical), 1.0,
                                             rgba.data_ptr(), L.stream_ptr()))
        return {'output': rgba, 'net_input': net_input}
