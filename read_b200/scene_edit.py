"""Scene editing and stitching: place several fitted scenes in one world, carve objects out of them, move, hide and instance
those objects, and render the result in ONE rasterizer pass (``ops.SegmentedPoints`` + ``read_raster_project_segments``).

Model.  A *scene* is a cloud with its ``[1,8,N]`` descriptors and a placement ``P`` into the composed world; its points get the
global ids ``base + original id``, bases in the order scenes are added, and the composed descriptor table is the scenes' textures
concatenated in that order, so the descriptor gather runs unchanged over global ids.  An *object* is a set of a scene's points
carved out of the scene's static segment into a segment of its own with a transform ``M``; an *instance* is one more segment
over an object's rows with its own transform (the same points and descriptors drawn twice).  Every scene, object and instance
is one segment, at most ``ops.MAX_SEGMENTS`` (4096) in all.

Matrix rule (the parity contract the tests restate): the matrix of a segment for view ``total_m`` (``FrameRenderer.total_matrix``,
float32) is ``T = total_m @ P_scene @ M``, with ``M`` the identity for the static segment, the object's transform for an object
and the instance's for an instance; the product is formed in float64 and rounded ONCE to float32 (``segment_matrices``), so an
identity placement and transform give ``total_m`` bit for bit.  Rows act on column vectors, as in the kernel:
``c_i = row_i . (x, y, z, 1)``.

Edits.  ``set_transform`` and ``set_visible`` change a host-side 4x4 or one visibility flag and never touch point data; the
per-segment matrices and flags are kept in arrays, so a frame's host work (``segment_matrices``, the visibility bytes) is a few
vectorised numpy operations whatever the segment count.  Adding a scene, object or instance changes the layout; the store is rebuilt (points re-sorted per segment) the next time it
is asked for.  A scene hidden with ``set_visible`` hides its objects and instances too; hiding an object leaves its instances.
"""
import numpy as np
import torch

from . import ops
from . import point_views
from . import sprites
from .texture import PointTexture


def _mat4(m, what):
    a = np.asarray(m, dtype=np.float64)
    if a.shape != (4, 4) or not np.all(np.isfinite(a)):
        raise ValueError(f"read_b200: {what} must be a finite 4x4 matrix")
    return a.copy()


class _Handle:
    def __init__(self, kind, index):
        self.kind, self.index = kind, index

    def __repr__(self):
        return f"<{self.kind} {self.index}>"


class SceneComposer:
    def __init__(self, device=None, cell=0.25):
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.cell = float(cell)
        self._scenes = []        # dict(xyz, base, n, P, visible, objects=[object index])
        self._objects = []       # dict(scene, ids (original ids, int64), M, visible, instances=[instance index])
        self._instances = []     # dict(object, M, visible)
        self._activation = None
        self._tex = None         # composed PointTexture [1, 8, total]
        self._store = None       # ops.SegmentedPoints, rebuilt after a layout change
        self._segments = []      # per segment: (handle, scene index)
        self._scene_P = np.empty((0, 4, 4))            # [scenes, 4, 4] placements (mirror of the dicts' "P")
        self._scene_vis = np.empty((0,), dtype=bool)   # [scenes] flags (mirror of the dicts' "visible")
        # per segment of the built layout: scene index, M (identity for a scene's static part), is-a-scene, own flag
        self._seg_scene = np.empty((0,), dtype=np.int64)
        self._seg_M = np.empty((0, 4, 4))
        self._seg_is_scene = np.empty((0,), dtype=bool)
        self._seg_own_vis = np.empty((0,), dtype=bool)
        self._seg_of = {}        # (kind, index) of an object or instance -> its segment
        self._tables = {}        # composed [total, 4] attribute tables, built on first use after a scene is added
        self.total = 0

    # ------------------------------------------------------------------ layout
    def _check_segments(self, extra):
        n = len(self._scenes) + len(self._objects) + len(self._instances) + extra
        if n > ops.MAX_SEGMENTS:
            raise ValueError(f"read_b200: a composed scene holds at most {ops.MAX_SEGMENTS} segments (scenes + objects + instances)")

    def add_scene(self, xyz, texture, placement=None, point_sizes=None, colors=None, normals=None):
        """Add a cloud ``xyz`` [N,3] with its descriptors (``[1,8,N]`` tensor or ``PointTexture``) and an optional 4x4
        ``placement`` into the composed world.  Returns the scene's handle; its points' global ids are ``handle.base + id``.
        ``point_sizes``: optional [N] per-point sprite sizes (read_b200.sprites), shared by the scene's objects and instances.
        ``colors`` / ``normals``: optional [N,3] per-point attributes for ``SceneRenderer.render_points``, shared likewise."""
        n = int(xyz.shape[0])
        sizes = None if point_sizes is None else sprites.check_point_sizes(point_sizes, n)
        attrs = {k: None if v is None else point_views.attribute_table(v, n, k, self.device)
                 for k, v in (("colors", colors), ("normals", normals))}
        if self.total + n >= 1 << 31:
            raise ValueError(f"read_b200: a composed scene of {self.total + n} points is too large; point ids must stay below 2^31")
        activation = texture.activation if isinstance(texture, PointTexture) else 'none'
        tex = texture.texture_ if isinstance(texture, PointTexture) else texture
        tex = torch.as_tensor(tex)
        if tex.dim() != 3 or tex.shape[0] != 1 or tex.shape[2] != n:
            raise ValueError(f"read_b200: the texture must be [1, D, {n}], got {tuple(tex.shape)}")
        if tex.shape[1] != 8:
            raise ValueError(f"read_b200: composed scenes use D = 8 descriptors, got D = {tex.shape[1]}")
        if self._activation is not None and activation != self._activation:
            raise ValueError(f"read_b200: every scene of a composition needs one activation ({self._activation!r}, got "
                             f"{activation!r})")
        P = _mat4(np.eye(4) if placement is None else placement, "placement")
        self._check_segments(1)
        xyz = torch.as_tensor(np.asarray(xyz, dtype=np.float32) if not torch.is_tensor(xyz) else xyz, dtype=torch.float32)
        if xyz.dim() != 2 or xyz.shape[1] != 3:
            raise ValueError("read_b200: in_points must be [N,3]")
        self._activation = activation
        h = _Handle("scene", len(self._scenes))
        h.base = self.total
        self._scenes.append(dict(xyz=xyz.to(self.device).contiguous(), base=self.total, n=n, P=P, visible=True, objects=[],
                                 sizes=None if sizes is None else sizes.to(self.device), **attrs))
        self._tables = {}
        self._scene_P = np.concatenate([self._scene_P, P[None]])
        self._scene_vis = np.append(self._scene_vis, True)
        self.total += n
        t = tex.detach().to(self.device, torch.float32)
        cat = t if self._tex is None else torch.cat([self._tex.texture_.detach(), t], 2)
        self._tex = PointTexture(8, 0, activation=activation)
        self._tex.texture_ = torch.nn.Parameter(cat.contiguous(), requires_grad=False)
        self._store = None
        return h

    def add_object(self, scene, point_ids, transform=None):
        """Carve the scene's points ``point_ids`` (original ids of that scene) into an object with its own 4x4 ``transform``
        (default identity).  A point belongs to at most one object."""
        sc = self._scene(scene)
        ids = torch.as_tensor(np.asarray(point_ids) if not torch.is_tensor(point_ids) else point_ids).to(torch.int64).reshape(-1).cpu()
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= sc["n"]):
            raise ValueError("read_b200: object point ids must be ids of the scene's points")
        if torch.unique(ids).numel() != ids.numel():
            raise ValueError("read_b200: an object lists a point twice")
        owned = [self._objects[o]["ids"] for o in sc["objects"]]
        if owned and bool(torch.isin(ids, torch.cat(owned)).any()):
            raise ValueError("read_b200: a point belongs to at most one object; these ids overlap another object")
        M = _mat4(np.eye(4) if transform is None else transform, "transform")
        self._check_segments(1)
        h = _Handle("object", len(self._objects))
        self._objects.append(dict(scene=scene.index, ids=ids, M=M, visible=True, instances=[]))
        sc["objects"].append(h.index)
        self._store = None
        return h

    def add_instance(self, obj, transform):
        """One more copy of object ``obj`` drawn with its own 4x4 ``transform``: a segment over the SAME rows (no point or
        descriptor is copied; the instance's pixels carry the object's global ids)."""
        return self.add_instances(obj, _mat4(transform, "transform")[None])[0]

    def add_instances(self, obj, transforms):
        """K more copies of object ``obj`` at once, one per 4x4 of ``transforms`` [K,4,4]: the same as K ``add_instance`` calls
        (handles in order), with one layout change."""
        ob = self._object(obj)
        T = np.asarray(transforms, dtype=np.float64)
        if T.ndim != 3 or T.shape[1:] != (4, 4) or not np.all(np.isfinite(T)):
            raise ValueError("read_b200: transforms must be finite [K, 4, 4] matrices")
        self._check_segments(T.shape[0])
        handles = []
        for M in T:
            h = _Handle("instance", len(self._instances))
            self._instances.append(dict(object=obj.index, M=M.copy(), visible=True))
            ob["instances"].append(h.index)
            handles.append(h)
        if handles:
            self._store = None
        return handles

    # ------------------------------------------------------------------ O(1) edits
    def _scene(self, h):
        if not isinstance(h, _Handle) or h.kind != "scene" or not 0 <= h.index < len(self._scenes):
            raise ValueError(f"read_b200: not a scene handle of this composer: {h!r}")
        return self._scenes[h.index]

    def _object(self, h):
        if not isinstance(h, _Handle) or h.kind != "object" or not 0 <= h.index < len(self._objects):
            raise ValueError(f"read_b200: not an object handle of this composer: {h!r}")
        return self._objects[h.index]

    def _entry(self, h):
        if isinstance(h, _Handle) and h.kind == "instance" and 0 <= h.index < len(self._instances):
            return self._instances[h.index]
        return self._scene(h) if isinstance(h, _Handle) and h.kind == "scene" else self._object(h)

    def set_transform(self, handle, M):
        """A scene's placement, an object's or an instance's transform (4x4).  Host-side only: takes effect on the next frame."""
        e = self._entry(handle)
        M = _mat4(M, "transform")
        if handle.kind == "scene":
            e["P"] = M
            self._scene_P[handle.index] = M
        else:
            e["M"] = M
            seg = self._seg_of.get((handle.kind, handle.index)) if self._store is not None else None
            if seg is not None:
                self._seg_M[seg] = M

    def set_visible(self, handle, visible):
        """Show or hide a scene (with its objects and instances), an object or an instance: one flag, no point data moves."""
        self._entry(handle)["visible"] = bool(visible)
        if handle.kind == "scene":
            self._scene_vis[handle.index] = bool(visible)
        if self._store is not None:
            if handle.kind != "scene":
                self._seg_own_vis[self._seg_of[(handle.kind, handle.index)]] = bool(visible)
            self._apply_visibility()

    # ------------------------------------------------------------------ what the renderer reads
    @property
    def texture(self):
        """The composed descriptors: a PointTexture over all global ids (scene textures concatenated in order)."""
        if self._tex is None:
            raise ValueError("read_b200: the composition holds no scene")
        return self._tex

    @property
    def colors(self):
        """The scenes' colours as one [total, 4] f32 table in global-id order (zeros for a scene without), or None if no scene
        has colours."""
        return self._table("colors")

    @property
    def normals(self):
        """The scenes' normals, as ``colors``."""
        return self._table("normals")

    def _table(self, name):
        if name not in self._tables:
            parts = [sc[name] for sc in self._scenes]
            self._tables[name] = None if all(p is None for p in parts) else torch.cat(
                [torch.zeros((sc["n"], 4), dtype=torch.float32, device=self.device) if p is None else p
                 for sc, p in zip(self._scenes, parts)])
        return self._tables[name]

    @property
    def store(self):
        """The ops.SegmentedPoints store of the current layout (rebuilt only after add_scene / add_object / add_instance)."""
        if self._store is None:
            self._build()
        return self._store

    def _build(self):
        if not self._scenes:
            raise ValueError("read_b200: the composition holds no scene")
        parts, segments, self._segments = [], [], []
        obj_part = {}
        for si, sc in enumerate(self._scenes):
            keep = torch.ones(sc["n"], dtype=torch.bool)
            for o in sc["objects"]:
                keep[self._objects[o]["ids"]] = False
            static = torch.nonzero(keep).reshape(-1)
            for ids in [static] + [self._objects[o]["ids"] for o in sc["objects"]]:
                dev_ids = ids.to(self.device)
                parts.append((sc["xyz"][dev_ids], dev_ids + sc["base"], None if sc["sizes"] is None else sc["sizes"][dev_ids]))
            segments.append(len(parts) - 1 - len(sc["objects"]))
            self._segments.append((_Handle("scene", si), si))
            for j, o in enumerate(sc["objects"]):
                obj_part[o] = len(parts) - len(sc["objects"]) + j
                segments.append(obj_part[o])
                self._segments.append((_Handle("object", o), si))
        for o, ob in enumerate(self._objects):
            for i in ob["instances"]:
                segments.append(obj_part[o])
                self._segments.append((_Handle("instance", i), ob["scene"]))
        self._store = ops.SegmentedPoints(parts, segments, n_ids=self.total, cell=self.cell)
        self._seg_scene = np.array([si for _, si in self._segments], dtype=np.int64)
        self._seg_is_scene = np.array([h.kind == "scene" for h, _ in self._segments], dtype=bool)
        self._seg_M = np.stack([np.eye(4) if h.kind == "scene" else self._entry(h)["M"] for h, _ in self._segments])
        self._seg_own_vis = np.array([h.kind == "scene" or self._entry(h)["visible"] for h, _ in self._segments], dtype=bool)
        self._seg_of = {(h.kind, h.index): s for s, (h, _) in enumerate(self._segments) if h.kind != "scene"}
        self._apply_visibility()

    def _apply_visibility(self):
        # a segment is drawn when its scene is shown and (for an object or instance) its own flag is set
        self._store.visible_flags().copy_(torch.from_numpy(self._scene_vis[self._seg_scene] & self._seg_own_vis))

    def segment_transforms(self):
        """[nseg, 4, 4] float64: P_scene @ M of every segment, in the store's segment order (a scene's static part: P itself)."""
        if self._store is None:
            self._build()
        P = self._scene_P[self._seg_scene]
        out = np.matmul(P, self._seg_M)
        out[self._seg_is_scene] = P[self._seg_is_scene]
        return out

    def segment_matrices(self, total_m):
        """The matrix rule: total_m [B,4,4] (or [4,4]) float32 -> seg_m [nseg, B, 4, 4] float32, T = total_m @ P @ M formed in
        float64 and rounded once."""
        return segment_matrices(total_m, self.segment_transforms())


def segment_matrices(total_m, transforms):
    """T[s, b] = total_m[b] @ transforms[s] in float64, rounded once to float32.  total_m [B,4,4] or [4,4] float32 (its values are
    used exactly), transforms [nseg,4,4]."""
    t = np.asarray(total_m, dtype=np.float32).reshape(-1, 4, 4).astype(np.float64)[None, :, :, :, None]    # [1,B,4,4,1]
    m = np.asarray(transforms, dtype=np.float64)[:, None, None, :, :]                                      # [S,1,1,4,4]
    acc = t[:, :, :, 0] * m[:, :, :, 0]                      # sum over j of t[b,i,j] * m[s,j,k], j = 0..3 in order
    for j in range(1, 4):
        acc = acc + t[:, :, :, j] * m[:, :, :, j]
    return acc.astype(np.float32)
