"""Point sprites: the point sizes of the reference's input-format keys and of a scene's ``point_sizes`` (DESIGN.md §4.2).

A key of ``input_format`` (``READ/gl/dataset.py:63-69``) names its point size with its LAST match of ``ps<N>`` or ``p<N>``:
``uv_1d_p3_ds1`` draws 3x3-pixel points, ``uv_1d_ps8`` draws points of ``max(1, 8 / c2)`` pixels (``c2`` the clip-space z, so
near points are larger), and a key without either is ``p1``.  Key ``l`` is pyramid level ``l``.  A per-point size ``s > 0``
replaces the key's ``N`` in either form; ``s == 0`` keeps it.  The rasterizer draws the levels of one frame in one pass
(``ops.raster_project_sprites``)."""
import re

import numpy as np
import torch

from . import _lib as L

MAX_POINT_SIZE = L.MAX_POINT_SIZE


def parse_point_size(key):
    """(N, relative) of one input-format key: the last ``ps\\d+`` / ``p\\d+`` match (relative for ``ps``), (1, False) without one."""
    res = re.findall('ps[0-9]+|p[0-9]+', key)
    if not res:
        return 1, False
    last = res[-1]
    return int(re.search('[0-9]+', last).group()), last.startswith('ps')


def sprite_levels(input_format, n_levels):
    """[(N, relative)] for the first ``n_levels`` keys of ``input_format`` (a comma-separated string or a list of keys).  Raises
    ValueError, naming the key, for a key that is not a ``uv`` key, a size of 0 or above ``MAX_POINT_SIZE``, or a ``_dsK`` whose K
    is not the key's position."""
    keys = input_format.replace(' ', '').split(',') if isinstance(input_format, str) else [str(k) for k in input_format]
    if len(keys) < n_levels:
        raise ValueError(f"read_b200: input_format {input_format!r} has {len(keys)} keys, {n_levels} levels need as many")
    out = []
    for l, key in enumerate(keys[:n_levels]):
        if not re.search('^uv', key):
            raise ValueError(f"read_b200: point sprites draw 'uv' keys only, not {key!r}")
        n, rel = parse_point_size(key)
        if n == 0:
            raise ValueError(f"read_b200: {key!r}: a point size of 0")
        if n > MAX_POINT_SIZE:
            raise ValueError(f"read_b200: {key!r}: point size {n} above the largest, {MAX_POINT_SIZE}")
        ds = re.findall('ds[0-5]+', key)
        if ds and int(ds[-1][2:]) != l:
            raise ValueError(f"read_b200: {key!r} is key {l} (level {l}) but names level {int(ds[-1][2:])}")
        out.append((n, rel))
    return out


def one_pixel(levels, point_sizes=None):
    """True when every level draws 1-pixel points: the rasterizer's existing path serves it."""
    return point_sizes is None and all(n == 1 and not rel for n, rel in levels)


def check_point_sizes(sizes, n):
    """``sizes`` ([n] array or tensor, any float dtype) as a float32 CPU tensor; ValueError for a length other than ``n`` and for
    negative, NaN or infinite sizes."""
    t = (sizes.detach() if torch.is_tensor(sizes) else torch.as_tensor(np.asarray(sizes))).to('cpu', torch.float32)
    if t.dim() != 1 or t.shape[0] != n:
        raise ValueError(f"read_b200: point_sizes must hold one size per point ({n}), got shape {tuple(t.shape)}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError("read_b200: point_sizes must be finite (no NaN or inf)")
    if bool((t < 0).any()):
        raise ValueError("read_b200: point_sizes must not be negative")
    return t.contiguous()


def desc(levels, point_sizes=None):
    """The C ABI's read_sprite_desc for ``levels`` [(N, relative)] and a device size column (or None)."""
    d = L.ReadSpriteDesc()
    for l, (n, rel) in enumerate(levels):
        d.size[l] = float(n)
        d.relative[l] = 1 if rel else 0
    d.point_sizes = None if point_sizes is None else point_sizes.data_ptr()
    return d
