"""Edge point sets for the rasterizer's exact tests (numpy only): points planted on the projection's edges, the matrices that
place them, hand-laid ring stores and a float32 restatement of the per-point projection.

Points reach clip space through one of two matrix forms:
  * per-view w (``view_matrix``): rows (1,0,0,0), (0,1,0,0), (0,0,1,m23), (0,0,0,w) give c = (x, y, z, w), so the points choose
    cx, cy, cz freely and every w class is a view of its own.  Points are normalized coordinates times w (``view_set``).
  * per-point w with a fixed cz (``point_matrix``): points (a*w, b*w, w) and rows (1,0,0,0), (0,1,0,0), (0,0,c,0), (0,0,1,0) give
    c = (a*w, b*w, fl(c*w), w), so one warp can mix denominators inside and outside the shared-reciprocal range.

The classes (labels per point): E1 frustum planes, E2 denominators, E3 depth, E4 pixel boundaries, E5 tiny quotients, E6 depth ties,
E7 sprites.  tests/test_raster_edges_host.py proves each planted value bit for bit with the kernel's own float32 arithmetic."""
import numpy as np

from scene_scale_util import clip_coords

F32 = np.float32
CHUNK = 1024                      # rows per ring chunk (RT_CHUNK)
BLOCK = 128                       # rows one compute warp of a ring chunk takes: 128 * k + 32 * u + lane, u = 0..3
ID_STALL = 0xFFFFFFFF             # an id word the ring never sees: a warp whose lane-0 ids are all ~0 would not free its stage


def up(x, k=1):
    x = F32(x)
    for _ in range(k):
        x = np.nextafter(x, F32(np.inf))
    return F32(x)


def down(x, k=1):
    x = F32(x)
    for _ in range(k):
        x = np.nextafter(x, F32(-np.inf))
    return F32(x)


def p2(e):
    return F32(2.0 ** e)


ONE_M, ONE_P = down(1.0), up(1.0)                 # one float32 ulp inside / outside a plane at 1
FLT_MAX = np.finfo(F32).max
SAFE_LO, SAFE_HI = p2(-57), p2(58)                # div_safe_den accepts |w| in [2^-57, 2^58): biased exponents 70 .. 184
DENORM = p2(-140)


def bits(x):
    return np.asarray(x, F32).view(np.uint32)


def div_safe(w):
    """raster.cu's div_safe_den: the biased exponent of |w| lies in [70, 184]."""
    u = (bits(w) & np.uint32(0x7FFFFFFF)).astype(np.uint64)
    return ((u - (70 << 23)) & 0xFFFFFFFF) < (115 << 23)


def view_matrix(w, m23=0.0):
    m = np.zeros((4, 4), F32)
    m[0, 0] = m[1, 1] = m[2, 2] = 1
    m[2, 3] = m23
    m[3, 3] = w
    return m


def point_matrix(c):
    m = np.zeros((4, 4), F32)
    m[0, 0] = m[1, 1] = 1
    m[2, 2] = c
    m[3, 2] = 1
    return m


def project(m, xyz, W, H):
    """The oracle's per-point projection in float32 (numpy float32 operations are correctly rounded): clip coordinates, IEEE
    quotients, the literal frustum test, d, u, v and the centre pixel.  vis: drawn at 1 pixel (NaN and d == 0 never are)."""
    c = clip_coords(m, xyz)
    with np.errstate(all="ignore"):
        q = (c[:, :3] / c[:, 3:4]).astype(F32)
        ok = ~np.isnan(q).any(1) & (np.abs(q) <= 1).all(1)
        d = ((q[:, 2] + F32(1)) * F32(0.5)).astype(F32)
        u = ((F32(W) * (q[:, 0] + F32(1))) * F32(0.5)).astype(F32)
        v = ((F32(H) * (F32(1) - q[:, 1])) * F32(0.5)).astype(F32)
        ok &= d != 0
        xx = np.where(ok, u, 0).astype(np.int64)
        yy = np.where(ok, v, 0).astype(np.int64)
    return {"c": c, "q": q, "d": d, "u": u, "v": v, "xx": xx, "yy": yy, "in": ok, "vis": ok & (xx < W) & (yy < H)}


def clip_in(m, xyz):
    """clip_point's division-free test |c_i| <= |c_3| (the ring's vote ignores rows that fail it)."""
    c = clip_coords(m, xyz)
    aw = np.abs(c[:, 3])
    with np.errstate(invalid="ignore"):
        return (np.abs(c[:, :3]) <= aw[:, None]).all(1)


def boundary_targets(n):
    """Pixel boundaries j of an n-pixel axis the sets plant: the ends, the middle, and multiples of n's odd part (where
    2j/n - 1 is a float whose u is exactly j for any n)."""
    odd = n
    while odd % 2 == 0:
        odd //= 2
    return sorted({0, 1, n // 2 - 1, n // 2, n // 2 + 1, n - 1, n, odd * max(1, n // (4 * odd)), n - odd * max(1, n // (4 * odd))})


def _ordered(x):
    """float32 -> an integer of the same order."""
    b = int(bits(F32(x)))
    return b if b < 0x80000000 else -(b & 0x7FFFFFFF)


def _unordered(k):
    return (np.array([k if k >= 0 else (-k) | 0x80000000], np.uint64).astype(np.uint32)).view(F32)[0]


def boundary_first(n, j):
    """The smallest float x in [-1, 1] whose u = fl(fl(n * fl(x + 1)) * 0.5) is at least j (u is monotonic in x): x gives pixel j,
    the float below it pixel j - 1."""
    lo, hi = _ordered(F32(-1)), _ordered(F32(1))
    while lo < hi:
        mid = (lo + hi) // 2
        if pixel_u(n, _unordered(mid)) >= j:
            hi = mid
        else:
            lo = mid + 1
    return _unordered(lo)


def boundary_x(n, j):
    """The float x whose u is exactly j, or None (no float lands exactly on this boundary)."""
    x = boundary_first(n, j)
    return x if pixel_u(n, x) == j else None


def boundary_coords(n):
    """Normalized coordinates at the pixel boundaries of an n-pixel axis: per target j the first float of pixel j and the floats
    either side of it, inside [-1, 1].  A y coordinate is the negation: 1 - (-x) and 1 + x round alike, so v = u."""
    out = []
    for j in boundary_targets(n):
        x0 = boundary_first(n, j)
        out += [down(x0), x0, up(x0)]
    return np.unique(np.clip(np.array(out, F32), F32(-1), F32(1)))


def pixel_u(n, x):
    """u = fl(fl(n * fl(x + 1)) * 0.5) in float32."""
    x = np.asarray(x, F32)
    return ((F32(n) * (x + F32(1))) * F32(0.5)).astype(F32)


def slot_collisions(W, H, groups=3):
    """Lean mode 3's filter slot (idx ^ idx >> 11) & 2047 of pixel idx = yy * W + xx: `groups` pairs of distinct pixels sharing a
    slot, as (xx, yy) pairs."""
    idx = np.arange(W * H, dtype=np.int64)
    slot = (idx ^ (idx >> 11)) & 2047
    out, seen = [], {}
    for i in idx[2048::97]:                                       # every slot is taken once among the first 2048 pixels
        a, b = int(np.nonzero(slot == slot[i])[0][0]), int(i)
        if slot[i] not in seen and a != b:
            seen[slot[i]] = b
            out.append(((a % W, a // W), (b % W, b // W)))
            if len(out) == groups:
                break
    return out


def centre(n, j, flip=False):
    """The normalized coordinate of pixel j's centre on an n-pixel axis (exact for power-of-two n); flip: the y axis."""
    x = F32((2.0 * j + 1.0) / n - 1.0)
    return -x if flip else x


def normalized_rows(W, H):
    """(A [n,3] f32, labels): normalized clip coordinates (cx, cy, cz) of the per-view-w classes at level 0 of W x H."""
    rows, lab = [], []

    def add(r, cls):
        rows.append([F32(v) for v in r])
        lab.append(cls)

    base = (F32(0.25), F32(-0.375), F32(0.5))
    for i in range(3):                                            # E1: each plane, one ulp inside and outside
        for s in (1, -1):
            for e, tag in ((F32(1), "on"), (ONE_M, "inside"), (ONE_P, "outside")):
                r = list(base)
                r[i] = F32(s) * e
                add(r, f"E1 plane c{i}={'+' if s > 0 else '-'}w {tag}")
    corner = (F32(-1), ONE_M * F32(-1), F32(0.5), ONE_M, F32(1))
    for x in corner:                                              # E1: edges and corners of the clip cube
        for y in corner:
            for z in (F32(1), ONE_M, F32(0.5), F32(-0.5)):
                add((x, y, z), "E1 edge/corner")
    for k in range(5):                                            # E3: d = 0 and the first four floats above it
        add((F32(-0.75 + 0.3 * k), F32(0.125), F32(-1.0 + k * 2.0 ** -24)), f"E3 cz=-1+{k}ulp")
    for z, tag in ((F32(1), "cz=1"), (ONE_M, "cz=1-ulp"), (F32(0), "cz=0")):
        add((F32(0.625), F32(0.375), z), f"E3 {tag}")
    cy0, cx0 = centre(H, 3, True), centre(W, 5)
    for i, x in enumerate(boundary_coords(W)):                    # E4: pixel boundaries, u = j exactly and the floats around it
        add((x, cy0, F32(0.5) - F32(i) * F32(2.0 ** -10)), "E4 u boundary")
    for i, y in enumerate(-boundary_coords(H)):
        add((cx0, y, F32(0.25) - F32(i) * F32(2.0 ** -10)), "E4 v boundary")
    add((F32(1), cy0, F32(0.5)), "E4 cx=1 (u=W)")
    add((cx0, F32(-1), F32(0.5)), "E4 cy=-1 (v=H)")
    for k, (cx, cy) in enumerate(((centre(W, 1), centre(H, 2, True)), (centre(W, W - 2), centre(H, H - 1, True)),
                                  (centre(W, W // 2), centre(H, 0, True)))):
        for _ in range(6):                                        # E6: identical keys but the id
            add((cx, cy, F32(0.125 * k)), "E6 tie")
    for (a, b) in slot_collisions(W, H):                          # E6: distinct pixels, one lean-mode-3 slot
        for (px, py), z in ((a, 0.3), (b, 0.2), (a, 0.25), (b, 0.1), (a, 0.25), (a, 0.35)):
            add((centre(W, px), centre(H, py, True), F32(z)), "E6 slot")
    return np.array(rows, F32).reshape(-1, 3), lab


TINY = (p2(-149), p2(-140), p2(-126), up(p2(-126)))


def tiny_rows():
    """E5: raw numerators down to 2^-149 (quotients in the denormal range for w in the safe range)."""
    rows = []
    for i, t in enumerate(TINY):
        for s in (1, -1):
            rows.append([F32(s) * t, F32(-s) * TINY[(i + 1) % 4], F32(s) * TINY[(i + 2) % 4]])
    rows.append([F32(0), TINY[0], F32(0)])
    return np.array(rows, F32)


# per-view w classes: (label, w)
VIEW_W = [("w=1", F32(1)), ("w=-1", F32(-1)), ("w=2^-57", SAFE_LO), ("w=pred(2^-57)", down(SAFE_LO)), ("w=-2^-57", -SAFE_LO),
          ("w=2^57", p2(57)), ("w=pred(2^58)", down(SAFE_HI)), ("w=2^58", SAFE_HI), ("w=-pred(2^58)", -down(SAFE_HI)),
          ("w=+0", F32(0)), ("w=-0", F32(-0.0)), ("w=2^-140", DENORM), ("w=FLT_MAX", FLT_MAX), ("w=+inf", F32(np.inf)),
          ("w=-inf", F32(-np.inf)), ("w=2^20", p2(20)), ("w=2^-20", p2(-20))]


def view_set(W, H):
    """The per-view-w set at level 0 of W x H: (xyz [n,3] f32 in id order, labels [n], matrices [len(VIEW_W),4,4]).  The
    normalized rows once unscaled and then times every finite non-zero w; the tiny numerators; (0,0,0) and nonzero numerators
    over w = 0."""
    A, lab = normalized_rows(W, H)
    xs, labels = [A], [f"raw {c}" for c in lab]
    t = tiny_rows()
    xs.append(t)
    labels += ["E5 tiny numerator"] * len(t)
    z = np.array([[0, 0, 0], [0.5, 0, 0], [0, -0.25, 0], [0, 0, 0.75], [-0.0, -0.0, -0.0]], F32)
    xs.append(z)
    labels += ["E2 zero or nonzero numerator over w=0"] * len(z)
    with np.errstate(over="ignore"):
        for name, w in VIEW_W:
            if w == 0 or not np.isfinite(w) or name == "w=1":
                continue
            xs.append((A * w).astype(F32))
            labels += [f"{name}: {c}" for c in lab]
    M = np.stack([view_matrix(w) for _, w in VIEW_W])
    return np.concatenate(xs).astype(F32), labels, M


# fixed cz of the per-point-w views: c such that cz = fl(fl(c * w) / w) sits near -1 (every bit of the quotient shows in d),
# d = 0 (c = -1), the far plane and ordinary depths
C_VALUES = [F32(-1 + 2.0 ** -24), F32(-1 + 2.0 ** -23), F32(-1 + 3 * 2.0 ** -24), F32(-1 + 2.0 ** -22), F32(-1), F32(1),
            F32(0.25), ONE_M]


def safe_ws(rng, n):
    """n random denominators in the shared-reciprocal range, both signs, random mantissas, exponents -57 .. 57."""
    m = rng.integers(1 << 23, 1 << 24, n).astype(np.float64) / (1 << 23)
    e = rng.integers(-57, 58, n)
    s = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    return (s * m * np.exp2(e)).astype(F32)


UNSAFE_VISIBLE = [FLT_MAX, DENORM, -FLT_MAX, -DENORM]            # visible rows the shared reciprocal would get wrong
UNSAFE_ALL = [F32(0), F32(-0.0), DENORM, p2(-149), down(SAFE_LO), SAFE_HI, -SAFE_HI, p2(100), FLT_MAX, -FLT_MAX]


def _coeffs(rng, n, W):
    """a or b of per-point rows: planes, one ulp either side, pixel boundaries and random values in [-1, 1]."""
    pool = np.concatenate([np.array([1, -1, ONE_M, -ONE_M, ONE_P, -ONE_P, 0], F32), boundary_coords(W),
                           rng.uniform(-1, 1, 64).astype(F32)])
    return pool[rng.integers(0, len(pool), n)]


def block_rows(rng, kind, W, H):
    """128 per-point-w rows (a, b, w) and labels for one block kind."""
    a, b = _coeffs(rng, BLOCK, W), _coeffs(rng, BLOCK, H)
    w = safe_ws(rng, BLOCK)
    lab = ["safe"] * BLOCK
    spot = {"unsafe_lane0": 0, "unsafe_lane31": 31, "unsafe_u3": 96 + 17, "unsafe_culled": 45}.get(kind)
    if kind.startswith("unsafe_") and kind != "unsafe_culled":
        w[spot] = UNSAFE_VISIBLE[spot % len(UNSAFE_VISIBLE)]
        a[spot], b[spot] = F32(0.625), F32(-0.4375)
        lab[spot] = "E2 visible unsafe w"
    elif kind == "unsafe_culled":
        w[spot] = FLT_MAX
        a[spot], b[spot] = F32(0.5), F32(1.5)                     # |b w| > |w|: culled before the vote
        lab[spot] = "E2 culled unsafe w"
    elif kind == "all_unsafe":
        w = np.array([UNSAFE_ALL[i % len(UNSAFE_ALL)] for i in range(BLOCK)], F32)
        lab = ["E2 unsafe w"] * BLOCK
    elif kind == "ties":
        a[:], b[:], w[:] = F32(0.25), F32(0.25), F32(1)
        lab = ["E6 tie"] * BLOCK
    return a, b, w, lab


def point_rows(a, b, w):
    """(a*w, b*w, w) in float32."""
    with np.errstate(all="ignore"):
        return np.stack([(a * w).astype(F32), (b * w).astype(F32), w.astype(F32)], 1)


BLOCK_KINDS = ["safe", "unsafe_lane0", "unsafe_lane31", "unsafe_u3", "unsafe_culled", "all_unsafe", "safe", "ties"]


def ring_store(W, H, seed=0, chunks=3, tail=333):
    """A hand-laid whole store of per-point-w rows: `chunks` chunks of the 8 BLOCK_KINDS (rotated per chunk, so each kind meets
    several compute warps) and a partial last chunk of `tail` rows.  Returns dict(xyz [n,3] in id order, ids [n] (row -> id),
    pts4 [n,4] (rows: x, y, z, id bits), labels [n] per id, kinds [per full block]).  Ties carry descending ids along the rows:
    higher ids in lower lanes, across warps and across chunks."""
    check_level0(W, H)
    rng = np.random.default_rng(seed)
    rows, lab, kinds = [], [], []
    for c in range(chunks):
        for k in range(CHUNK // BLOCK):
            kind = BLOCK_KINDS[(k + c) % len(BLOCK_KINDS)]
            a, b, w, l = block_rows(rng, kind, W, H)
            rows.append(point_rows(a, b, w))
            lab += l
            kinds.append(kind)
    a, b, w, l = block_rows(rng, "safe", W, H)
    rows.append(point_rows(a[:tail], b[:tail], w[:tail]))
    lab += l[:tail]
    r = np.concatenate(rows)
    n = r.shape[0]
    ids = rng.permutation(n).astype(np.int64)
    tie = np.array([x == "E6 tie" for x in lab])
    ids[tie] = np.sort(ids[tie])[::-1]                            # descending along the rows
    xyz = np.empty_like(r)
    xyz[ids] = r
    labels = [""] * n
    for row, i in enumerate(ids):
        labels[i] = lab[row]
    return {"xyz": xyz, "ids": ids, "pts4": pts4_of(r, ids), "labels": labels, "kinds": kinds, "W": W, "H": H}


def pts4_of(rows, ids):
    """[n,4] f32 store rows: (x, y, z, id bits).  Asserts the ring's safety rule: no id word 0xFFFFFFFF."""
    ids = np.asarray(ids, np.int64)
    assert ids.min(initial=0) >= 0 and ids.max(initial=0) < ID_STALL, "an id word of 0xFFFFFFFF would stall the ring"
    out = np.empty((rows.shape[0], 4), F32)
    out[:, :3] = rows
    out[:, 3] = ids.astype(np.uint32).view(F32)
    return out


def check_level0(W, H):
    """The ring kernels index level 0 with 32 bits."""
    assert W * H < 2 ** 31, "level 0 must stay below 2^31 pixels"


def lay_segments(parts, seed=0):
    """Lay parts out as a segmented store.  parts: [(xyz [m,3] in local id order, labels [m], sizes [m] or None)].  Each part's rows
    are a random permutation of its points, padded to whole chunks with (NaN, NaN, NaN, id 0); global id = the part's base + local
    id, so global ids increase with local ids and a per-part oracle z-buffer maps to global keys by adding the base.  Returns
    dict(pts4, psize (per row, 0 for padding; None without sizes), parts [(first_chunk, chunks, xyz, id base, sizes)], labels per
    global id)."""
    rng = np.random.default_rng(seed)
    sized = any(p[2] is not None for p in parts)
    blocks, sizes, meta, labels, first, gid = [], [], [], [], 0, 0
    for xyz, lab, sz in parts:
        m = xyz.shape[0]
        local = rng.permutation(m)                                 # row -> local id
        rows = -(-m // CHUNK) * CHUNK
        blk = np.zeros((rows, 4), F32)
        blk[m:, :3] = np.nan
        blk[:m] = pts4_of(xyz[local], gid + local)
        blocks.append(blk)
        if sized:
            col = np.zeros(rows, F32)
            if sz is not None:
                col[:m] = sz[local]
            sizes.append(col)
        meta.append((first, rows // CHUNK, xyz, gid, sz))
        labels += list(lab)
        first += rows // CHUNK
        gid += m
    pts4 = np.concatenate(blocks)
    assert bits(pts4[:, 3]).max() < ID_STALL
    return {"pts4": pts4, "psize": np.concatenate(sizes) if sized else None, "parts": meta, "labels": labels}


def segmented_store(W, H, seed=1):
    """The segmented store of the ring tests: a part of mixed safe / unsafe per-point-w rows, and parts whose chunk boxes touch the
    x = w plane from inside (a in [1/2, 1], some a == 1, w = 1), lie just outside it (a from 1 + ulp) and far outside it."""
    check_level0(W, H)
    rng = np.random.default_rng(seed)
    parts = []
    got = [block_rows(rng, k, W, H) for k in ("unsafe_lane0", "all_unsafe", "safe", "unsafe_u3")]
    a, b, w = (np.concatenate([g[i] for g in got]) for i in range(3))
    parts.append((point_rows(a, b, w), sum((g[3] for g in got), []), None))
    n = 700
    ones = np.ones(n, F32)
    a = rng.uniform(0.5, 1.0, n).astype(F32)
    a[:3] = F32(1)                                                # the box's hi x is exactly w
    for a, tag in ((a, "inside"), (np.linspace(float(ONE_P), 1.25, n).astype(F32), "just outside"),
                   (rng.uniform(2, 3, n).astype(F32), "far outside")):
        parts.append((point_rows(a, rng.uniform(-1, 1, n).astype(F32), ones), [f"box {tag} x=w"] * n, None))
    return lay_segments(parts, seed)


# sprite classes: per-point sizes (E7) and the level sets the sprite tests draw
SPRITE_SIZES = [("nan", F32(np.nan)), ("negative", F32(-3)), ("denormal", DENORM), ("+inf", F32(np.inf)), ("0 (level N)", F32(0)),
                ("0.5", F32(0.5)), ("pred(0.5)", down(0.5)), ("1.5", F32(1.5)), ("2", F32(2)), ("2.5", F32(2.5)),
                ("63.5", F32(63.5)), ("pred(63.5)", down(63.5)), ("64", F32(64)), ("64.5", F32(64.5)), ("1e30", F32(1e30))]


def sprite_set(W, H):
    """Sprite edge points for per-view w = 1 with m23 = -0 (so c2 = -0 survives the dot product): (xyz [n,3], labels, sizes [n]).
    Relative sizes meet c2 = +0, -0, negative and denormal; even widths meet u - xx = 0.5 exactly and the floats either side;
    sprites sit at the corners and edges of the level so their squares cross all four borders."""
    rows, lab = [], []
    for z, tag in ((F32(0), "c2=+0"), (F32(-0.0), "c2=-0"), (F32(-0.5), "c2<0"), (DENORM, "c2 denormal"),
                   (-DENORM, "c2 -denormal"), (F32(0.5), "c2=0.5"), (ONE_M, "c2=1-ulp")):
        rows.append((F32(-0.375), F32(-0.625), z))                 # x, y < 0: x*0 and y*0 are -0, so c2 = -0 for z = -0
        lab.append(f"E7 relative {tag}")
    x5, y3 = centre(W, 5), centre(H, 3, True)
    for x in (down(x5), x5, up(x5)):                               # even widths: u - xx = 0.5 exactly and either side
        for y in (down(y3), y3, up(y3)):
            rows.append((x, y, F32(0.3)))
            lab.append("E7 half-pixel centre")
    last = F32(1 - 2.0 ** -22)                                      # 1 + last < 2: u just below W (ONE_M + 1 rounds to 2: dropped)
    for x in (F32(-1), -ONE_M, F32(0), ONE_M, last):               # the four borders and corners
        for y in (-last, -ONE_M, F32(0), ONE_M, F32(1)):
            rows.append((x, y, F32(0.6)))
            lab.append("E7 border")
    xyz = np.array(rows, F32)
    n = xyz.shape[0]
    # every size on every class, one copy per size (a copy shadows the later ones only where its square is drawn)
    xs = np.concatenate([xyz] * len(SPRITE_SIZES))
    labels = [f"{l}, size {name}" for name, _ in SPRITE_SIZES for l in lab]
    sz = np.concatenate([np.full(n, s, F32) for _, s in SPRITE_SIZES])
    return xs, labels, sz
