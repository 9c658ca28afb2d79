"""Drop-in for ``READ.models.compose.NetAndTexture`` (READ/models/compose.py:84-181) and ``ModelAndLoss`` (compose.py:12-32).

Contract kept (what train.py, viewer.py and READ/gl/nn.py:76-129 rely on):

* constructor ``(net, textures, supersampling=1, temporal_average=False)``; attributes ``net``, ``ss``, ``temporal_average``,
  ``last_input`` are poked from outside (nn.py:100-103);
* textures are parked on the CPU and become sub-modules (named by their id) only between ``load_textures`` / ``unload_textures``,
  so ``.cuda()``, ``.parameters()`` and ``state_dict()`` see exactly the loaded scenes; ``reg_loss`` sums over them;
* ``forward(inputs_dict)``: dict of index maps keyed by format string (every key containing 'uv' is sampled by the item's texture,
  the keys that follow it are concatenated in front of the samples) + ``'id'``; returns ``[B,3,H,W]`` (and, with
  ``return_input=True``, the LAST item's multi-scale net input, as the reference's loop leaves it).

Eval-mode batches run as ONE batched net pass (equivalent under eval-mode BatchNorm, SURVEY.md §8a "Batching"); in training mode
the reference's per-item loop is kept, because BatchNorm statistics are per call there, unless the net normalises each item on its
own (``UNet.train_batchnorm = 'per_item'``): then one batched pass computes what the loop does.  A batch that mixes scenes takes
the batched pass too, its items sampling their own textures in one gather (``_texture_table`` says when); otherwise it keeps the
loop.

Extra fast path (not in the reference): ``render(points, total_m, W, H)`` goes points -> packed z-buffer pyramid -> feature
pyramid -> net without materialising index maps, including the viewer's ``supersampling`` and ``temporal_average`` options.
"""
import functools

import torch
import torch.nn as nn

from . import ops
from . import panorama as pano_mod
from . import sprites
from . import _lib as L
from .texture import PointTexture, sample_items


def _as_id_list(texture_ids):
    if torch.is_tensor(texture_ids):
        return [int(t) for t in texture_ids.cpu().reshape(-1).tolist()]
    if isinstance(texture_ids, int):
        return [texture_ids]
    return [int(t) for t in texture_ids]


class NetAndTexture(nn.Module):
    def __init__(self, net, textures, supersampling=1, temporal_average=False):
        super().__init__()
        self.net = net
        self.ss = supersampling
        self.temporal_average = temporal_average
        self.last_input = None
        if not hasattr(textures, 'items'):
            try:
                textures = dict(textures)
            except TypeError:                       # a single texture module
                textures = {0: textures}
        self._textures = {tid: tex.cpu() for tid, tex in textures.items()}        # parked until loaded
        self._loaded_textures = []
        self._fused = {}                             # state of the fused path: pyramid, staging buffers, temporal history
        self._fused_pano = {}                        # the same for panoramas, so frames and panoramas keep their own histories

    # ------------------------------------------------------------------ texture residency (compose.py:102-123)
    def load_textures(self, texture_ids):
        ids = texture_ids.cpu().tolist() if torch.is_tensor(texture_ids) else (
            [texture_ids] if isinstance(texture_ids, int) else texture_ids)
        for tid in ids:
            self.add_module(str(tid), self._textures[tid])
        self._loaded_textures = ids

    def unload_textures(self):
        for tid in self._loaded_textures:
            name = str(tid)
            self._modules[name].cpu()
            del self._modules[name]

    def _texture(self, tid):
        return self._modules[str(tid)]

    def reg_loss(self):
        return sum((self._texture(tid).reg_loss() for tid in self._loaded_textures), 0)

    # ------------------------------------------------------------------ index-map path
    def _multiscale_input(self, texture, item):
        """One net input per 'uv' key: [extra channels that follow the key ..., texture samples], reduced by 1/ss when
        supersampling (compose.py:143-165).  ``texture``: the module (or any callable) that samples a 'uv' map."""
        keys = list(item)
        assert 'uv' in keys[0], 'first input must be uv'
        groups = []                                   # [(uv key, [extra keys])]
        for k in keys:
            if 'uv' in k:
                groups.append((k, []))
            else:
                groups[-1][1].append(k)
        scales = []
        for uv_key, extra in groups:
            parts = [item[k] for k in extra] + [texture(item[uv_key])]
            x = parts[0] if len(parts) == 1 else torch.cat(parts, 1)
            if self.ss > 1:
                x = nn.functional.interpolate(x, scale_factor=1. / self.ss, mode='bilinear')
            scales.append(x)
        return scales

    def _texture_table(self, texture_ids):
        """(textures, slots) for ONE net call over a batch whose items use two or more textures (item b samples
        ``textures[slots[b]]``, texture.sample_items), or None when the batch keeps the per-item loop: the textures must be
        PointTextures with 8 channels on one device, with one activation and one gradient mode (requires_grad, sparse or dense),
        at most 16 of them for at most 64 items."""
        distinct = list(dict.fromkeys(texture_ids))
        if not 2 <= len(distinct) <= L.MAX_TEX_SLOTS or len(texture_ids) > L.MAX_TEX_ITEMS:
            return None
        textures = [self._texture(tid) for tid in distinct]
        if not all(isinstance(t, PointTexture) and t.texture_.dim() == 3 and t.texture_.shape[1] == 8 for t in textures):
            return None
        if (len({t.activation for t in textures}) != 1 or len({t.texture_.device for t in textures}) != 1
                or len({(t.texture_.requires_grad, bool(getattr(t, '_sparse_requested', False))) for t in textures}) != 1):
            return None
        slot = {tid: s for s, tid in enumerate(distinct)}
        return textures, [slot[tid] for tid in texture_ids]

    def _direct_engine_forward(self, maps, texture_ids):
        """Inference shortcut of the index-map surface (VERDICT r01 #12): four 'uv' maps and nothing else, no supersampling /
        temporal average / autograd -> the descriptors are gathered from the index maps STRAIGHT into the engine's NHWC inputs
        (same values as PointTexture.forward followed by the engine's NCHW f32 -> NHWC conversion: both round the same f32 sample
        once) and the net runs; items of different scenes read their own textures in the same launch.  Returns None when the call
        does not qualify."""
        net = self.net
        if (self.ss != 1 or self.temporal_average or net.training or getattr(net, '_is_replica', False)
                or len(maps) != 4 or not all('uv' in k for k in maps)):
            return None
        if len(set(texture_ids)) == 1:
            textures, slots = [self._texture(texture_ids[0])], None
        else:
            table = self._texture_table(texture_ids)
            if table is None:
                return None
            textures, slots = table
        if not all(isinstance(t, PointTexture) and t.texture_.is_cuda and t.texture_.shape[1] == 8 for t in textures):
            return None
        if torch.is_grad_enabled() and (any(t.texture_.requires_grad for t in textures)
                                        or any(p.requires_grad for p in net.parameters())):
            return None
        vals = list(maps.values())
        B, _, H, W = vals[0].shape
        if len(texture_ids) != B or H % 16 or W % 16 or any(tuple(v.shape) != (B, 1, H >> l, W >> l) for l, v in enumerate(vals)):
            return None
        tex = textures[0]
        dev = tex.texture_.device
        eng = net.engine(B, H, W, dev)
        layout = L.FEAT_NHWC_BF16 if eng.bf16 else L.FEAT_NHWC_F32
        nds = [t.point_major() for t in textures]
        for l, v in enumerate(vals):
            ids = ops.index_map(v[:, 0], dev)
            if slots is None:
                ops.gather_from_index(nds[0], ids, layout, tex.activation, out=eng.inputs[l])
            else:
                ops.gather_from_index_items(nds, slots, ids, layout, tex.activation, out=eng.inputs[l])
        return eng.run().clone()

    def forward(self, inputs, **kwargs):
        maps = {k: v for k, v in inputs.items() if k != 'id'}
        texture_ids = _as_id_list(inputs['id'])
        if not kwargs:
            out = self._direct_engine_forward(maps, texture_ids)
            if out is not None:
                return out
        one_texture = len(set(texture_ids)) == 1
        items_apart = not self.net.training or getattr(self.net, 'train_batchnorm', 'batch') == 'per_item'
        batchable = len(texture_ids) > 1 and not self.temporal_average and items_apart
        table = None if one_texture or not batchable else self._texture_table(texture_ids)
        if batchable and (one_texture or table is not None):
            # eval-mode BatchNorm is per-pixel affine, and per-item train-mode BatchNorm normalises each item with its own
            # statistics: B batch-1 passes == one batch-B pass; items of different scenes sample their own textures in one gather
            sample = self._texture(texture_ids[0]) if one_texture else functools.partial(sample_items, *table)
            net_input = self._multiscale_input(sample, maps)
            out = self.net(*net_input, **kwargs)
            net_input = [t[-1:] for t in net_input]              # the reference returns the last item's input
        else:
            frames = []
            for i, tid in enumerate(texture_ids):                # compose.py:136
                net_input = self._multiscale_input(self._texture(tid), {k: v[i][None] for k, v in maps.items()})
                if self.temporal_average:
                    if self.last_input is not None:
                        net_input = [(cur + prev) / 2 for cur, prev in zip(net_input, self.last_input)]
                    self.last_input = list(net_input)
                frames.append(self.net(*net_input, **kwargs))
            out = torch.cat(frames, 0)
        return (out, net_input) if kwargs.get('return_input') else out

    # ------------------------------------------------------------------ fused fast path
    def _fused_state(self, B, Wr, Hr, n_levels, device, staged, Hn, Wn, st=None):
        st = self._fused if st is None else st
        key = (B, Wr, Hr, n_levels, str(device), staged, Hn, Wn)
        if st.get('key') != key:
            st.clear()
            st['key'] = key
            st['pyr'] = ops.Pyramid(B, Wr, Hr, n_levels, device)
            st['clean'] = False
            if staged:
                st['feat'] = [torch.empty((B, Hr >> l, Wr >> l, 8), dtype=torch.float32, device=device) for l in range(4)]
                st['last'] = [torch.empty((B, Hn >> l, Wn >> l, 8), dtype=torch.float32, device=device) for l in range(4)]
                st['have_last'] = False
        return st

    @torch.no_grad()
    def render(self, xyz, total_m, W, H, texture_id=0, n_levels=4, want_maps=False, return_input=False, clone_output=True,
               seg_visible=None, input_format=None, panorama=None):
        """points [N,3] (cuda f32) or an ``ops.SortedPoints`` store + total_m [B,4,4] (cuda f32) -> RGB [B,3,H,W] f32 (a fresh
        tensor), all on device, one pass over the cloud.  A sorted store serves frames whose levels nest; the result is
        bit-identical to rendering the unsorted cloud (the z-buffer is a min over (depth | original id) keys).

        ``self.ss`` > 1 renders the pyramid at ss x (W, H) and reduces every level's features bilinearly, ``temporal_average``
        blends each level with the previous frame's (already blended) input - both exactly as ``forward`` does on index maps.
        ``want_maps``: also return the (index, depth) maps per level, index maps of ``ops.index_map_dtype(N)`` (float32 up to
        2^24 + 1 points, int32 above); ``return_input``: also return the net input
        (list of [B,8,h,w] f32, the reference's ``net_input``); ``clone_output=False`` hands out the engine's own output buffer
        (valid until the next frame) for callers that consume it immediately.

        An ``ops.SegmentedPoints`` store (read_b200.scene_edit) takes ``total_m`` as the per-segment matrices ``seg_m``
        [nseg, B, 4, 4]; its index maps hold global ids, which index the composed texture.  It is drawn by the culled rasterizer
        (``ops.raster_project_segments_culled``): only the chunks that are visible and may meet some view's frustum are read.
        ``seg_visible``: its [nseg] uint8 visibility flags already on the device (default: the store's host flags).

        ``input_format``: the checkpoint's format string; its first ``n_levels`` keys give each level's point size (``_pN`` /
        ``_psN``, read_b200.sprites), and a store's per-point sizes (``psize``) apply.  Frames with larger points are drawn as point
        sprites from the store (SortedPoints or SegmentedPoints, whose levels need not nest) and gathered level by level;
        ``None`` (the default), or only 1-pixel levels and no per-point sizes, renders as without it.

        ``panorama``: a ``read_b200.panorama.Panorama`` of ``W`` x ``H`` pixels, drawn from a store (SortedPoints or
        SegmentedPoints) with ``total_m`` the world -> camera matrices (``Panorama.world_to_camera``; per segment for a segmented
        store).  The pyramid and the net run at (W + 2 margin) x H, the result is the [B,3,H,W] crop without the margins;
        ``want_maps`` and ``return_input`` give the full width, margins included.  Panoramas keep a temporal history of their own,
        apart from the frames'.  Point sprites raise ValueError."""
        segmented = isinstance(xyz, ops.SegmentedPoints)
        store = xyz if segmented or isinstance(xyz, ops.SortedPoints) else None
        pts = store.pts4 if store is not None else xyz
        n_ids = store.n_ids if segmented else (store.n if store is not None else pts.shape[0])
        map_dtype = ops.index_map_dtype(n_ids)                  # ValueError at 2^31 points or more
        L.require_device()
        lib = L.load()
        texture = self._texture(texture_id)
        B = total_m.shape[1] if segmented else total_m.shape[0]
        ss = int(self.ss)
        if panorama is not None:
            if store is None:
                raise ValueError("read_b200: panoramas are drawn from an ops.SortedPoints or ops.SegmentedPoints store")
            if (W, H) != (panorama.width, panorama.height):
                raise ValueError(f"read_b200: W, H = {W}, {H} for a {panorama!r}")
            margin = panorama.margin
            W = panorama.plane_width                            # the pyramid and the net run with the margins
        Wr, Hr = W * ss, H * ss
        eng = self.net.engine(B, H, W, pts.device)
        staged = ss > 1 or bool(self.temporal_average)
        st = self._fused_state(B, Wr, Hr, n_levels, pts.device, staged, H, W,
                               None if panorama is None else self._fused_pano)
        pyr = st['pyr']
        if not self.temporal_average:
            st['have_last'] = False
        tex = texture.point_major()
        act_layout = L.FEAT_NHWC_BF16 if eng.bf16 else L.FEAT_NHWC_F32
        gather_layout = L.FEAT_NHWC_F32 if staged else act_layout
        gather_out = st['feat'] if staged else eng.inputs
        levels = None if input_format is None else sprites.sprite_levels(input_format, n_levels)
        sprite = levels is not None and not sprites.one_pixel(levels, store.psize if store is not None else None)
        if sprite and store is None:
            raise ValueError("read_b200: point sprites are drawn from an ops.SortedPoints or ops.SegmentedPoints store")
        if sprite and panorama is not None:
            raise ValueError("read_b200: panoramas draw 1-pixel points; point sprites (_pN / _psN keys, per-point sizes) are "
                             "drawn on frames only")
        fused_ok = (not sprite and not want_maps and texture.activation == 'none'
                    and ops.fused_resolve_supported(pyr, tex.shape[1]))

        if not (fused_ok and st['clean']):
            pyr.clear()
        if panorama is not None:
            pr = panorama.scaled(ss)
            if segmented:
                pano_mod.raster_panorama_segments_culled(pyr, store, total_m, pr, seg_visible)
            else:
                pano_mod.raster_panorama_sorted(pyr, store, total_m, pr)
            if not fused_ok:
                ops.raster_derive(pyr)
        elif sprite:
            ops.raster_project_sprites(pyr, store, total_m, levels, visible=seg_visible)
        elif store is not None:
            if pyr.direct_mask != 1:
                raise RuntimeError("a SortedPoints store renders frames with nested levels; pass the [N,3] cloud otherwise")
            if segmented:
                ops.raster_project_segments_culled(pyr, store, total_m, seg_visible)
            else:
                ops.raster_project_sorted(pyr, store, total_m)
            if not fused_ok:
                ops.raster_derive(pyr)
        else:
            ops.raster_project(pyr, pts, total_m, derive=not fused_ok)
        if fused_ok:
            # ONE kernel derives levels 1..3, gathers the four feature maps and leaves level 0 cleared for the next frame
            ops.pyramid_resolve_gather(tex, pyr, gather_out, gather_layout, reset_level0=True)
        else:
            for l in range(4):
                ops.gather_from_zbuf(tex, pyr, l, gather_layout, texture.activation, out=gather_out[l])
        st['clean'] = fused_ok
        if staged:
            sp = L.stream_ptr()
            for l in range(4):
                last = st['last'][l] if self.temporal_average else None
                L.check(lib.read_stage_net_inputs(st['feat'][l].data_ptr(), B, Hr >> l, Wr >> l, 8, ss, L.ptr(last),
                                                  int(st['have_last']), eng.act_code, eng.inputs[l].data_ptr(), sp))
            st['have_last'] = bool(self.temporal_average)
        out = eng.run()
        if panorama is not None and margin:
            out = out[..., margin:W - margin].contiguous()       # a fresh tensor without the wrapped columns
        elif clone_output:                   # the engine's output buffer is reused by the next frame
            out = out.clone()
        extras = []
        if want_maps:
            extras.append([ops.zbuf_resolve(pyr, l, index_dtype=map_dtype) for l in range(n_levels)])
        if return_input:
            extras.append([ops.nhwc_to_nchw(t) for t in eng.inputs])
        return (out, *extras) if extras else out


class ModelAndLoss(nn.Module):
    """The wrapper train.py puts under nn.DataParallel so that model AND criterion are scattered (compose.py:12-32): positional
    arguments are (model inputs ..., target); returns ``(output, loss)``; an optional ``mask`` kwarg multiplies the output
    before the loss when ``use_mask`` is set."""

    def __init__(self, model, loss, use_mask=False):
        super().__init__()
        self.model, self.loss, self.use_mask = model, loss, use_mask

    def forward(self, *args, **kwargs):
        *model_inputs, target = args
        output = self.model(*model_inputs, **kwargs)
        mask = kwargs.get('mask') if self.use_mask else None
        loss = self.loss(output if mask is None else output * mask, target)
        return output, loss
