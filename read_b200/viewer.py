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
from . import point_views
from . import sprites
from .compose import NetAndTexture
from .texture import PointTexture
from .unet import UNet


def _panorama_result(out, panorama, flip_vertical, net_input):
    """``infer``'s result for a panorama: the displayable [H,W,4] surface of the net's [1,3,H,W] crop (alpha 1, flipped with
    ``flip_vertical``) and the net input."""
    H, W = panorama.height, panorama.width
    rgba = torch.empty((H, W, 4), dtype=torch.float32, device=out.device)
    L.check(L.load().read_frame_to_rgba(out.data_ptr(), H, W, int(flip_vertical), 1.0, rgba.data_ptr(), L.stream_ptr()))
    return {'output': rgba, 'net_input': net_input}


class FrameRenderer:
    def __init__(self, xyz, net_state_dict, texture, viewport_size, supersampling=1, temporal_average=False,
                 device=None, flip_vertical=False, n_levels=4, return_net_input=True, input_format=None, point_sizes=None,
                 colors=None, normals=None):
        """xyz: [N,3] float32 (numpy / tensor); net_state_dict: UNet checkpoint ``state_dict``; texture: the
        ``[1,8,N]`` descriptor tensor (``PointTexture.texture_``) or a ``PointTexture``; viewport_size: (W, H) of the output
        frame.  ``supersampling`` / ``temporal_average``: the options of READ/gl/nn.py:76,100-103 (the pyramid is rendered at
        ss x the viewport and reduced bilinearly; every level is averaged with the previous frame's input), served on the fused
        path.  ``return_net_input=False`` skips materialising the reference's ``net_input`` list (4 small transposes).
        ``input_format``: the checkpoint's format string (``args.input_format``); its first ``n_levels`` keys' ``_pN`` / ``_psN``
        point sizes are drawn as point sprites (read_b200.sprites).  ``point_sizes``: optional [N] per-point sizes (the scene's
        ``point_sizes``), which replace the keys' sizes where > 0; without ``input_format`` every level is a ``_p1`` key.
        ``colors`` / ``normals``: optional [N,3] per-point colours (``scene_data['pointcloud']['rgb']``) and normals, the
        attributes ``render_points`` draws; uploaded once."""
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
        if point_sizes is not None and input_format is None:
            input_format = ','.join(['uv_1d'] * n_levels)
        self.input_format = input_format
        levels = None if input_format is None else sprites.sprite_levels(input_format, n_levels)
        sprite = levels is not None and not sprites.one_pixel(levels, point_sizes)
        # point sprites are drawn from the sorted store whatever the level sizes
        self.store = ops.SortedPoints(self.xyz, point_sizes=point_sizes) if nested or sprite else None
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
        n = self.xyz.shape[0]
        self.colors = None if colors is None else point_views.attribute_table(colors, n, "colors", self.device)
        self.normals = None if normals is None else point_views.attribute_table(normals, n, "normals", self.device)
        self._views = point_views.ViewState(W, H, self.device)
        self._points_store = None          # sorted store for point-sprite views when the frame path keeps none
        self._bounds = None

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
                                    n_levels=self.n_levels, return_input=self.return_net_input, clone_output=False,
                                    input_format=self.input_format)
        out, net_input = res if self.return_net_input else (res, None)                       # out: [1,3,H,W] f32
        rgba = torch.empty((self.H, self.W, 4), dtype=torch.float32, device=self.device)
        L.check(L.load().read_frame_to_rgba(out.data_ptr(), self.H, self.W, int(self.flip_vertical), 1.0,
                                             rgba.data_ptr(), L.stream_ptr()))
        return {'output': rgba, 'net_input': net_input}

    def infer_panorama(self, view_matrix, panorama):
        """A cylindrical panorama (read_b200.panorama.Panorama) from the camera ``view_matrix`` (camera-to-world, GL convention):
        -> {'output': [H,W,4] f32 cuda tensor, 'net_input': the four [1,8,h,w] net inputs at the rendered width, margins
        included (None with ``return_net_input=False``)}, as ``infer``.  Drawn from the sorted store (built here once if the
        frame path keeps none); its temporal history is kept apart from ``infer``'s.  Point sprites raise ValueError."""
        store = self.store
        if store is None:
            if self._points_store is None:
                self._points_store = ops.SortedPoints(self.xyz)
            store = self._points_store
        m = self._upload_camera(panorama.world_to_camera(view_matrix))
        with torch.no_grad():
            res = self.model.render(store, m, panorama.width, panorama.height, n_levels=self.n_levels,
                                    return_input=self.return_net_input, clone_output=False, input_format=self.input_format,
                                    panorama=panorama)
        out, net_input = res if self.return_net_input else (res, None)
        return _panorama_result(out, panorama, self.flip_vertical, net_input)

    def render_points(self, proj_matrix, view_matrix, mode='color', submode=0, point_size=1, relative=False,
                      clear_color=(0., 0., 0., 1.)):
        """The reference viewer's point-cloud view (viewer.py:263-285): -> {'output': [H,W,4] f32 cuda tensor}, a fresh tensor whose
        rows are in ``infer``'s order (flipped the same way with ``flip_vertical``).  Each pixel shows its winning point (the
        z-buffer's minimum depth, ties to the lowest id) coloured by ``mode``: 'color' (the ``colors`` table), 'pca' (a 3-component
        PCA of the descriptors, ``--pca``), 'normals' (``submode`` 0..4: model, reflection, camera frame, view direction, raw),
        'depth' (clip-space z), 'uv' (submode 0: the point id), 'xyz' (position in the cloud's bounding box) or 'label' (normal x
        / 255); an empty pixel gets ``clear_color``.  ``point_size`` (1..64) and ``relative`` (size / clip z) draw point sprites
        with the scene's per-point sizes, as the frame path's ``_pN`` / ``_psN`` keys do; a per-point size of 0 keeps
        ``point_size`` (GL would draw such a point at size 0).  Arithmetic: include/read_b200.h, read_point_view."""
        clear = point_views.check_view_args(mode, submode, point_size, clear_color)
        table = point_views.table_for(mode, self.colors, self.normals,
                                      lambda: self._views.pca(self.model._texture(0).texture_))
        total = self.total_matrix(proj_matrix, view_matrix)
        m = self._upload_camera(total)
        pyr = self._views.pyramid()
        store = self.store
        with torch.no_grad():
            if point_size != 1 or relative or (store is not None and store.psize is not None):
                if store is None:
                    if self._points_store is None:
                        self._points_store = ops.SortedPoints(self.xyz)
                    store = self._points_store
                ops.raster_project_sprites(pyr, store, m, [(float(point_size), bool(relative))])
            elif store is not None:
                ops.raster_project_sorted(pyr, store, m)
            else:
                ops.raster_project(pyr, self.xyz, m)
            if mode == 'xyz' and self._bounds is None:
                self._bounds = (self.xyz.min(0).values.cpu().numpy(), self.xyz.max(0).values.cpu().numpy())
            lo, hi = self._bounds if mode == 'xyz' else ((0., 0., 0.), (0., 0., 0.))
            geometry = mode in ('normals', 'depth', 'xyz')
            out = point_views.shade(pyr, mode, submode, table, self.xyz if geometry else None, total, view_matrix, lo, hi,
                                    clear, self.flip_vertical)
        return {'output': out}


class SceneRenderer:
    """``FrameRenderer`` for a composed scene (read_b200.scene_edit.SceneComposer): several scenes, moved / hidden / instanced
    objects, all rendered in one rasterizer pass over the composer's segmented store.  ``infer`` keeps ``FrameRenderer.infer``'s
    contract exactly.  Edits made on the composer between two ``infer`` calls show in the second frame; a layout change (a scene,
    object or instance added) re-sorts the points once, a transform or visibility change moves no point data."""

    def __init__(self, composer, net_state_dict, viewport_size, supersampling=1, temporal_average=False, flip_vertical=False,
                 return_net_input=True, n_levels=4, input_format=None):
        """``input_format``: the checkpoint's format string, as for FrameRenderer; the scenes' ``point_sizes`` (SceneComposer.add_scene)
        apply with it.  Point-sprite frames need not have nested levels."""
        W, H = int(viewport_size[0]), int(viewport_size[1])
        assert W % 16 == 0, f'set width {16 * (W // 16)}'
        assert H % 16 == 0, f'set height {16 * (H // 16)}'
        assert int(supersampling) >= 1, 'supersampling must be a positive integer'
        self.device = composer.device
        L.require_device(self.device.index)
        ss = int(supersampling)
        self.input_format = input_format
        levels = None if input_format is None else sprites.sprite_levels(input_format, n_levels)
        if (levels is None or sprites.one_pixel(levels)) and L.load().read_raster_direct_mask(W * ss, H * ss, n_levels) != 1:
            raise ValueError("read_b200: a composed scene renders frames whose pyramid levels nest (each exactly half of the last)")
        self.composer = composer
        self.W, self.H, self.n_levels = W, H, n_levels
        self.flip_vertical = bool(flip_vertical)
        self.return_net_input = bool(return_net_input)
        net = UNet()
        net.load_state_dict(net_state_dict, strict=True)
        self._tex = composer.texture
        self.model = NetAndTexture(net, {0: self._tex}, ss, temporal_average=bool(temporal_average))
        self.model.load_textures(0)
        self.model.to(self.device).eval()
        # per frame, the [nseg, 1, 4, 4] matrices and the [nseg] visibility bytes in ONE copy, through a ring of pinned staging
        # buffers (see FrameRenderer._upload_camera)
        self._m_host = [torch.empty(ops.MAX_SEGMENTS * 65, dtype=torch.uint8).pin_memory() for _ in range(4)]
        self._m_used = [None] * 4
        self._m_i = 0
        self._views = point_views.ViewState(W, H, self.device)

    def _upload(self, seg_m, visible):
        """-> (seg_m, visible) on the device: [nseg, 1, 4, 4] f32 and [nseg] uint8."""
        i = self._m_i
        self._m_i = (i + 1) % len(self._m_host)
        if self._m_used[i] is not None:
            self._m_used[i].synchronize()                # the copy that last read this staging buffer (4 frames ago) has run
        nseg = seg_m.shape[0]
        host = self._m_host[i][:nseg * 65]
        host[:nseg * 64].view(torch.float32).copy_(torch.from_numpy(seg_m).reshape(-1))
        host[nseg * 64:].copy_(visible)
        dev = host.to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._m_used[i] = ev
        return dev[:nseg * 64].view(torch.float32).view(nseg, 1, 4, 4), dev[nseg * 64:]

    def infer(self, proj_matrix, view_matrix):
        """-> {'output': [H,W,4] f32 cuda tensor, 'net_input': list of the four [1,8,h,w] f32 net inputs (None with
        ``return_net_input=False``)}, as ``FrameRenderer.infer``; both fresh tensors."""
        comp = self.composer
        if comp.texture is not self._tex:                # a scene was added: the composed descriptor table grew
            self._tex = comp.texture
            self.model._textures[0] = self._tex
            self.model.add_module('0', self._tex.to(self.device))
        store = comp.store
        seg_m, visible = self._upload(comp.segment_matrices(FrameRenderer.total_matrix(proj_matrix, view_matrix)),
                                      store.visible_flags())
        with torch.no_grad():
            res = self.model.render(store, seg_m, self.W, self.H, n_levels=self.n_levels, return_input=self.return_net_input,
                                    clone_output=False, seg_visible=visible, input_format=self.input_format)
        out, net_input = res if self.return_net_input else (res, None)
        rgba = torch.empty((self.H, self.W, 4), dtype=torch.float32, device=self.device)
        L.check(L.load().read_frame_to_rgba(out.data_ptr(), self.H, self.W, int(self.flip_vertical), 1.0,
                                             rgba.data_ptr(), L.stream_ptr()))
        return {'output': rgba, 'net_input': net_input}

    def infer_panorama(self, view_matrix, panorama):
        """``FrameRenderer.infer_panorama`` for the composed scene: every segment drawn under
        ``composer.segment_matrices(Panorama.world_to_camera(view_matrix))``, units beyond ``zfar`` in every view culled."""
        comp = self.composer
        if comp.texture is not self._tex:                # a scene was added: the composed descriptor table grew
            self._tex = comp.texture
            self.model._textures[0] = self._tex
            self.model.add_module('0', self._tex.to(self.device))
        store = comp.store
        seg_m, visible = self._upload(comp.segment_matrices(panorama.world_to_camera(view_matrix)), store.visible_flags())
        with torch.no_grad():
            res = self.model.render(store, seg_m, panorama.width, panorama.height, n_levels=self.n_levels,
                                    return_input=self.return_net_input, clone_output=False, seg_visible=visible,
                                    input_format=self.input_format, panorama=panorama)
        out, net_input = res if self.return_net_input else (res, None)
        return _panorama_result(out, panorama, self.flip_vertical, net_input)

    def render_points(self, proj_matrix, view_matrix, mode='color', submode=0, point_size=1, relative=False,
                      clear_color=(0., 0., 0., 1.)):
        """``FrameRenderer.render_points`` for the composed scene, in the modes a pixel's id alone determines: 'color', 'pca' (over
        the composed descriptor table), 'uv' (the global id) and 'label', with the tables of ``SceneComposer.add_scene``
        concatenated in global-id order.  'normals', 'depth' and 'xyz' need the point's world position, which an instance's
        id does not give (every instance of an object carries the object's ids): they raise ValueError."""
        clear = point_views.check_view_args(mode, submode, point_size, clear_color)
        if mode not in point_views.ID_MODES:
            raise ValueError(f"read_b200: mode {mode!r} needs the point's world position, which a composed scene's ids do not "
                             f"identify; a composed scene draws the modes {point_views.ID_MODES}")
        comp = self.composer
        table = point_views.table_for(mode, comp.colors, comp.normals, lambda: self._views.pca(comp.texture.texture_))
        store = comp.store
        seg_m, visible = self._upload(comp.segment_matrices(FrameRenderer.total_matrix(proj_matrix, view_matrix)),
                                      store.visible_flags())
        pyr = self._views.pyramid()
        with torch.no_grad():
            if point_size != 1 or relative or store.psize is not None:
                ops.raster_project_sprites(pyr, store, seg_m, [(float(point_size), bool(relative))], visible=visible)
            else:
                ops.raster_project_segments_culled(pyr, store, seg_m, visible)
            out = point_views.shade(pyr, mode, submode, table, None, None, None, None, None, clear, self.flip_vertical)
        return {'output': out}
