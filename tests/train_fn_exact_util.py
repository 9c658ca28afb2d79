"""Per-element checks of the bf16 training autograd Function of read_b200/blocks.py (ConvChainFn, as stack_forward, gated_conv and
gated_conv_srcs call it, in every BatchNorm mode): a float64 replay of each call's launch sequence, the exact-tier operands and
their precondition, and the case lists; shared by test_train_fn_exact_host.py (no GPU) and test_gpu_train_fn_exact.py.

The replay follows the launches the Functions document and rounds to bf16 (round to nearest even) where they do:
  forward   x -> NHWC bf16 (nchw_to_nhwc); each conv's output bf16(A(f + b_f) * sigmoid(m + b_m) * scale + shift [+ residual]),
            the ResBlock skip added before that rounding (the conv epilogue's residual operand);
  backward  the output gradient -> NHWC bf16 (_out_grad); [f | m] recomputed by a RAW launch, bf16(f), bf16(m), the biases added
            in fp32; [df | dm] rounded to bf16 (the gate backward's output), dbias_f / dbias_m from the unrounded fp32 df / dm;
            dgamma = sum dy (g - mean) inv_std and dbeta = sum dy over every pixel; the weight gradient from the bf16 [df | dm]
            and the saved bf16 input (fp32 sums); the input gradient bf16(exact sum [+ the ResBlock skip gradient]), the skip
            added inside that rounding (dgrad's residual operand); a residual's gradient is the output gradient itself, not
            rounded.
The Functions run a conv with C < 16 padded to 16 and SCM*.main.3 (C = 56 / 120 / 248) padded to 64 / 128 / 256; padded channels
have zero filters, biases and scale / shift, so they compute 0, take a zero output gradient and their gradient rows are sliced
away: the replay runs the real channels only.  With ``R=ident`` every rounding is the identity and the replay is float64
autograd of the same GatedConv modules (test_train_fn_exact_host.py checks that on every case).

Exact tier (eval-mode BatchNorm).  Operands that make every stage exact, so each element has one correct value:
* every operand is an integer; the f filters are sparse; wm = 0 and
  bias_m = PIN_BIAS_M, so m + b_m = 64 at every pixel: sigmoid is exactly 1.0 in fp32 in the forward (fwd_exact_util) and in the
  gate backward (conv_bwd.cu: 1.f / (1.f + expf(-m)) with expf(-64) < 2^-90, so 1 + expf(-64) rounds to 1), and dm = dg * A * s
  * (1 - s) is exactly 0;
* an ELU conv's bias_f exceeds every |f| twice over, so f + b_f > 0 (the ELU is the identity) before and after f's bf16
  rounding; running_mean = bias_f re-centres it;
* eps = 0 and running_var = 1 fold BatchNorm exactly: scale = gamma, shift = beta - running_mean * gamma, all dyadic.
``precondition`` then proves, stage by stage on the replay's own values, that every fp32 sum a kernel forms (any order, any split)
is a multiple of its unit below 2^24 units: the sum of the terms' absolute values over their common unit (the product of the
operands' smallest power-of-two units).
"""
import dataclasses
import math
import zlib

import torch
import torch.nn.functional as F

import bwd_exact_util as U
import fwd_exact_util as X

EXACT_LIMIT = U.EXACT_LIMIT
PIN_BIAS_M = 64.0
NONREP_FLOOR = 0.05         # share of an exact case's output values that bf16 cannot hold
ROUND_FLOOR = 0.1           # per family, the same share at every rounding point in its best case
NAMES = ("dwf", "dbias_f", "dwm", "dbias_m", "dgamma", "dbeta")
NNZ = 2                     # nonzero f-filter taps per output channel (sparse: keeps an 8-conv stack's values exact)


# ---------------------------------------------------------------- cases
@dataclasses.dataclass(frozen=True)
class Case:
    """One Function call.  family: 'stack' (stack_forward, 8 convs at C = cin = cout), 'single' (gated_conv, 3x3 stride 1,
    optional residual) or 'multi' (gated_conv_srcs over ``srcs``, 1x1 or stride 2).  need: 'all', 'frozen' (no parameter
    needs a gradient) or 'no_x' (the input needs none)."""
    name: str
    family: str
    srcs: tuple
    cout: int
    k: int
    stride: int
    B: int
    H: int
    W: int
    elu: bool = True
    residual: bool = False
    need: str = "all"

    @property
    def cin(self):
        return sum(self.srcs)

    @property
    def pad(self):
        return (self.k - 1) // 2

    @property
    def id(self):
        return f"{self.family}-{self.name}-B{self.B}-{self.H}x{self.W}" + (f"-{self.need}" if self.need != "all" else "")

    @property
    def n_convs(self):
        return 8 if self.family == "stack" else 1

    def elus(self):
        return [i % 2 == 0 for i in range(8)] if self.family == "stack" else [self.elu]


def _stack(C, B, H, W, **kw):
    return Case(f"C{C}", "stack", (C,), C, 3, 1, B, H, W, **kw)


# stacks: C = 32 / 64 (weight-stationary bodies) and 128 / 256 (the role-swapped streamed-weight body, R = 16 on small
# images); B = 1, 2, 3; H, W multiples of none of 8, 16, 17; one pixel wide.  The large frozen / input-only cases reach R = 17
# on a 132-SM H100 (test_gpu_train_fn_exact.py asserts which R each case gets).
STACK_CASES = [
    _stack(32, 1, 11, 13), _stack(32, 3, 5, 1), _stack(64, 2, 7, 5), _stack(64, 1, 1, 19),
    _stack(128, 2, 5, 7), _stack(128, 1, 9, 1), _stack(256, 3, 3, 5), _stack(256, 1, 6, 3),
    _stack(256, 3, 33, 55, need="frozen"), _stack(128, 1, 33, 359, need="frozen"), _stack(64, 2, 13, 10, need="no_x"),
]
STACK_R = {(256, 3, 33, 55): 17, (128, 1, 33, 359): 17, (128, 2, 5, 7): 16, (128, 1, 9, 1): 16, (256, 3, 3, 5): 16,
           (256, 1, 6, 3): 16}


def _single(name, cin, cout, B, H, W, elu, residual=False, **kw):
    return Case(name, "single", (cin,), cout, 3, 1, B, H, W, elu=elu, residual=residual, **kw)


# single convs: every row of unet.layer_table they run (feat_extract.0 is the 8-channel dgrad_cin8 path, feat_extract.5 runs
# padded to 16, FAM*.merge with its residual)
SINGLE_CASES = [
    _single("feat_extract.0", 8, 32, 2, 9, 7, True),
    _single("feat_extract.5", 32, 3, 1, 11, 5, False),
    _single("SCM2.main.0", 8, 16, 3, 5, 3, True),
    _single("SCM1.main.0", 8, 32, 1, 7, 1, True),
    _single("SCM0.main.0", 8, 64, 2, 3, 5, True),
    _single("SCM2.main.2", 32, 32, 2, 5, 9, True),
    _single("SCM1.main.2", 64, 64, 1, 9, 5, True),
    _single("SCM0.main.2", 128, 128, 2, 3, 7, True),
    _single("AFFs.0.conv.1", 32, 32, 1, 13, 3, False),
    _single("AFFs.1.conv.1", 64, 64, 3, 3, 3, False),
    _single("AFFs.2.conv.1", 128, 128, 1, 5, 5, False),
    _single("FAM2.merge", 64, 64, 2, 5, 3, False, residual=True),
    _single("FAM1.merge", 128, 128, 1, 7, 3, False, residual=True),
    _single("FAM0.merge", 256, 256, 1, 3, 5, False, residual=True),
]


def _multi(name, srcs, cout, k, stride, B, H, W, elu, **kw):
    return Case(name, "multi", tuple(srcs), cout, k, stride, B, H, W, elu=elu, **kw)


# gated_conv_srcs: every 1x1 and stride-2 row.  AFFs.*.conv.0 read four sources (480 channels, the 256-channel one split into
# two 128-channel input-gradient parts); SCM*.main.3 runs padded (C = 56 / 120 / 248) and, at 120 / 248, recomputes [f | m] per
# 64-channel block; SCM0.conv has one 256-channel source; Convs.* read two sources of equal width.  Odd H, W for 1x1, even H, W
# that are not multiples of 16 for stride 2.
MULTI_CASES = [
    _multi("AFFs.0.conv.0", (32, 64, 128, 256), 32, 1, 1, 1, 5, 3, True),
    _multi("AFFs.1.conv.0", (32, 64, 128, 256), 64, 1, 1, 2, 3, 3, True),
    _multi("AFFs.2.conv.0", (32, 64, 128, 256), 128, 1, 1, 1, 3, 1, True),
    _multi("SCM2.main.1", (16,), 32, 1, 1, 2, 7, 5, True),
    _multi("SCM1.main.1", (32,), 64, 1, 1, 1, 9, 3, True),
    _multi("SCM0.main.1", (64,), 128, 1, 1, 3, 3, 3, True),
    _multi("SCM2.main.3", (32,), 56, 1, 1, 2, 5, 7, True),
    _multi("SCM1.main.3", (64,), 120, 1, 1, 1, 7, 5, True),
    _multi("SCM0.main.3", (128,), 248, 1, 1, 3, 3, 1, True),
    _multi("SCM2.conv", (64,), 64, 1, 1, 1, 9, 7, False),
    _multi("SCM1.conv", (128,), 128, 1, 1, 2, 3, 5, False),
    _multi("SCM0.conv", (256,), 256, 1, 1, 1, 5, 3, False),
    _multi("Convs.0", (128, 128), 128, 1, 1, 1, 5, 5, True),
    _multi("Convs.1", (64, 64), 64, 1, 1, 2, 3, 7, True),
    _multi("Convs.2", (32, 32), 32, 1, 1, 1, 11, 3, True),
    _multi("feat_extract.1", (32,), 64, 3, 2, 1, 10, 6, True),
    _multi("feat_extract.2", (64,), 128, 3, 2, 2, 6, 2, True),
    _multi("feat_extract.6", (128,), 256, 3, 2, 1, 6, 10, True),
    _multi("feat_extract.3", (128,), 64, 4, 2, 1, 14, 2, True),
    _multi("feat_extract.4", (64,), 32, 4, 2, 2, 6, 10, True),
    _multi("feat_extract.7", (256,), 128, 4, 2, 1, 2, 6, True),
]

EXACT_CASES = STACK_CASES + SINGLE_CASES + MULTI_CASES


# ---------------------------------------------------------------- modules and exact-tier operands
def _valuation(t):
    """log2 of the largest power of two dividing every element of the float64 tensor ``t`` (0 for an all-zero tensor)."""
    t = t.double()
    nz = t[t != 0]
    if nz.numel() == 0:
        return 0
    for e in range(-60, 60):
        if bool((torch.frac(nz * 2.0 ** -e) == 0).all()) is False:
            return e - 1
    return 59


def unit(t):
    return 2.0 ** _valuation(t)


def make_mods(case):
    """The case's GatedConv modules (real channel counts), default-initialised; the operands replace their parameters."""
    from read_b200.unet import GatedConv
    if case.family == "stack":
        return [GatedConv(case.cout, case.cout, 3, 1, e) for e in case.elus()]
    return [GatedConv(case.cin, case.cout, case.k, case.stride, case.elu)]


def _sparse_filters(cout, cin, k, gen, nnz, amp):
    """[cout, cin, k, k] integers in +-[1, amp], at least ``nnz`` per output channel; entry e = co * nnz + j sits at tap e mod k^2
    and in the 8-channel input block e mod (blocks), and nnz grows until cout * nnz reaches both counts, so every tap and every
    block holds nonzero filters."""
    w = torch.zeros((cout, cin, k * k))
    nblk = -(-cin // 8)
    nnz = max(nnz, -(-max(k * k, nblk) // cout))
    for co in range(cout):
        for j in range(nnz):
            e = co * nnz + j
            blk = e % nblk
            ci = 8 * blk + int(torch.randint(0, min(8, cin - 8 * blk), (1,), generator=gen))
            v = int(torch.randint(1, amp + 1, (1,), generator=gen)) * (1 if torch.rand(1, generator=gen) < 0.5 else -1)
            w[co, ci, e % (k * k)] = v
    return w.reshape(cout, cin, k, k)


def _pow2_ceil(v):
    return 2.0 ** math.ceil(math.log2(max(v, 1.0)))


def set_exact_params(mod, x, gen, stack):
    """Give ``mod`` exact-tier parameters for the NCHW float64 input ``x`` it will see (module docstring).  Every parameter is an
    integer, so every value of the chain is: a stack's convs have one filter tap of +-1 per output channel and gamma = +-1 (the
    values grow only through the skips), a lone conv two taps up to +-3 and gamma in {+-1, +-3} (so dy * gamma needs rounding)."""
    b = mod.block
    cout, cin, k, _ = b['conv_f'].weight.shape
    wf = _sparse_filters(cout, cin, k, gen, 1 if stack else 2, 1 if stack else 3)
    acc = F.conv2d(x, wf.double(), stride=mod.stride, padding=(k - 1) // 2)
    amax = float(acc.abs().max()) if acc.numel() else 1.0
    if mod.elu:
        bf = torch.full((cout,), 2 * _pow2_ceil(amax + 1))
        rm = bf.clone()
    else:
        bf = U.int_tensor((cout,), 64, gen, 0.2)
        rm = U.int_tensor((cout,), 64, gen, 0.2)
    gvals = torch.tensor([1.0, -1.0] if stack else [1.0, -1.0, 3.0, -3.0])
    gamma = gvals[torch.randint(0, len(gvals), (cout,), generator=gen)]
    beta = U.int_tensor((cout,), 32, gen, 0.2)
    with torch.no_grad():
        b['conv_f'].weight.copy_(wf)
        b['conv_f'].bias.copy_(bf)
        b['conv_m'].weight.zero_()
        b['conv_m'].bias.fill_(PIN_BIAS_M)
        n = b['norm']
        n.eps = 0.0
        n.weight.copy_(gamma)
        n.bias.copy_(beta)
        n.running_mean.copy_(rm)
        n.running_var.fill_(1.0)
    mod.eval()


def params64(mod):
    b = mod.block
    n = b['norm']
    p = {k: v.detach().double() for k, v in (("wf", b['conv_f'].weight), ("bf", b['conv_f'].bias), ("wm", b['conv_m'].weight),
                                              ("bm", b['conv_m'].bias), ("gamma", n.weight), ("beta", n.bias))}
    p["mean"], p["var"] = n.running_mean.detach().double(), n.running_var.detach().double()
    p["inv"] = 1.0 / torch.sqrt(p["var"] + n.eps)
    p["scale"] = p["gamma"] * p["inv"]
    p["shift"] = p["beta"] - p["mean"] * p["scale"]
    return p


def exact_operands(case, seed=0):
    """(modules, inputs NCHW float32, residual or None, output gradient NCHW float32) of an exact-tier case.  Inputs and the
    output gradient are integers; |output gradient| <= amp, where amp is the largest of 1023, 511, ... for which the case meets
    its precondition (the weight-gradient sums over every pixel bound it on the larger images)."""
    gen = torch.Generator().manual_seed(zlib.crc32(f"{case.id}/{seed}".encode()))
    mods = make_mods(case)
    xs = [U.int_tensor((case.B, c, case.H, case.W), 255, gen, 0.2) for c in case.srcs]
    res = U.int_tensor((case.B, case.cout, case.H, case.W), 255, gen, 0.2) if case.residual else None
    t = rnd(torch.cat(xs, 1).double())
    if case.family == "stack":
        for r in range(0, 8, 2):
            set_exact_params(mods[r], t, gen, True)
            h = _fwd_conv(t, params64(mods[r]), mods[r], None, rnd)[0]
            set_exact_params(mods[r + 1], h, gen, True)
            t = _fwd_conv(h, params64(mods[r + 1]), mods[r + 1], t, rnd)[0]
    else:
        set_exact_params(mods[0], t, gen, False)
    Ho, Wo = _out_hw(case)
    base = torch.randint(-1023, 1024, (case.B, case.cout, Ho, Wo), generator=gen).double()
    base = base * (torch.rand(base.shape, generator=gen) >= 0.2)
    for amp in (1023, 511, 255, 127, 63, 31, 15, 7, 3, 1):
        gout = torch.clamp(base, -amp, amp).float()
        try:
            precondition(case, mods, xs, res, gout)
            return mods, xs, res, gout
        except AssertionError:
            continue
    precondition(case, mods, xs, res, gout)
    return mods, xs, res, gout


def _out_hw(case):
    return ((case.H + 2 * case.pad - case.k) // case.stride + 1, (case.W + 2 * case.pad - case.k) // case.stride + 1)


# ---------------------------------------------------------------- the replay
def rnd(v):
    """bf16 round-to-nearest-even of float64 values that fp32 holds exactly (the precondition asserts it), back in float64."""
    return v.float().bfloat16().double()


def ident(v):
    return v


def _conv(x, w, mod):
    return F.conv2d(x, w, stride=mod.stride, padding=(mod.k - 1) // 2)


def _fwd_conv(x, p, mod, res, R):
    """(output, accf, accm, output before its rounding) of one gated conv in eval mode over the NCHW float64 input ``x``."""
    accf, accm = _conv(x, p["wf"], mod), _conv(x, p["wm"], mod)
    f, m = accf + p["bf"][:, None, None], accm + p["bm"][:, None, None]
    A = F.elu(f) if mod.elu else f
    y = A * torch.sigmoid(m) * p["scale"][:, None, None] + p["shift"][:, None, None]
    if res is not None:
        y = y + res
    return R(y), accf, accm, y


def _nhwc_rows(t):
    """NCHW [B, C, H, W] -> [B * H * W, C] (bwd_exact_util's pixel-row layout)."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _nchw(rows, like):
    B, _, H, W = like.shape
    return rows.reshape(B, H, W, -1).permute(0, 3, 1, 2)


def _gate(f_raw, m_raw, gy, p, elu, kind="eval", items=1, stats=None):
    """bwd_exact_util.gate_ref on NCHW operands: f_raw / m_raw are the RAW recompute (bias not added), gy the bf16 output
    gradient; ``stats`` (mean, inv, scale, s0, s1 [items, C]) replace the eval-mode fold of ``p``.  Returns gate_ref's dict and
    [df | dm] in concat order, NCHW."""
    C = f_raw.shape[1]
    # the RAW column order is defined for the channel counts the Functions run at: pad C = 120 / 248 to 128 / 256 with zero
    # output gradients (inv_std 1, everything else 0) and slice the results back
    Cp = 64 * -(-C // 64) if C > 64 else C
    padc = lambda t, v=0.0: torch.cat([t, torch.full(t.shape[:-1] + (Cp - C,), v, dtype=t.dtype)], -1)
    rows = lambda t: padc(_nhwc_rows(t))
    o = dict(fm=U.to_raw(torch.cat([rows(f_raw), rows(m_raw)], 1)), dy=rows(gy), bf=padc(p["bf"]), bm=padc(p["bm"]))
    st = stats if stats is not None else dict(scale=p["scale"][None], mean=p["mean"][None], inv=p["inv"][None])
    o.update({k: padc(v, 1.0 if k == "inv" else 0.0) for k, v in st.items()})
    n = o["dy"].shape[0]
    ref = U.gate_ref(o, Cp, elu, kind, items, n // items)
    for k in ("dfm", "T_dfm"):
        cat = torch.empty_like(ref[k])
        cat[:, U.fm_columns(Cp)] = ref[k]
        ref[k] = torch.cat([cat[:, :C], cat[:, Cp:Cp + C]], 1)         # concat order, real channels
    ref = {k: (v[..., :C] if k not in ("dfm", "T_dfm") else v) for k, v in ref.items()}
    return ref, _nchw(ref["dfm"][:, :C], gy), _nchw(ref["dfm"][:, C:], gy)


def _bwd_conv(x, p, mod, accf, accm, gy, skip, R, need_x):
    """The eval-mode backward of one gated conv: returns (dx or None, [dwf, dbf, dwm, dbm, dgamma, dbeta], stage values).  ``gy``
    is the bf16 output gradient, ``skip`` the gradient dgrad adds in its epilogue.  The gate / BatchNorm formulas are
    bwd_exact_util.gate_ref's."""
    ref, df, dm = _gate(R(accf), R(accm), gy, p, mod.elu)
    grads = [None, ref["sum_df"], None, ref["sum_dm"], ref["dgamma"], ref["dbeta"]]
    dfr, dmr = R(df), R(dm)
    pad = (mod.k - 1) // 2
    wshape = tuple(p["wf"].shape)
    grads[0] = torch.nn.grad.conv2d_weight(x, wshape, dfr, stride=mod.stride, padding=pad)
    grads[2] = torch.nn.grad.conv2d_weight(x, wshape, dmr, stride=mod.stride, padding=pad)
    dx = None
    if need_x:
        dsum = (torch.nn.grad.conv2d_input(tuple(x.shape), p["wf"], dfr, stride=mod.stride, padding=pad) +
                torch.nn.grad.conv2d_input(tuple(x.shape), p["wm"], dmr, stride=mod.stride, padding=pad))
        dx = dsum if skip is None else dsum + skip
    f = R(accf) + p["bf"][:, None, None]
    # with the gate pinned open and an ELU input positive (precondition) the gated value g is f itself
    st = dict(x=x, f=f, g=f, gy=gy, df=df, dfr=dfr, dmr=dmr, skip=skip)
    return dx, grads, st


def replay(case, mods, xs, res, gout, R=rnd):
    """Eval-mode forward and backward of the case's Function.  Returns dict(out, dxs (per source, None where not needed), dres,
    grads (6 per conv, in the Function's order), fwd / bwd (per conv stage values), pre (rounding point -> the exact values it
    rounds))."""
    need_x = case.need != "no_x"
    ts = [R(x.double()) for x in xs]
    t = torch.cat(ts, 1)
    ps = [params64(m) for m in mods]
    fwd = []
    if case.family == "stack":
        for r in range(0, 8, 2):
            h, af0, am0, hp = _fwd_conv(t, ps[r], mods[r], None, R)
            y, af1, am1, yp = _fwd_conv(h, ps[r + 1], mods[r + 1], t, R)
            fwd += [dict(x=t, accf=af0, accm=am0, res=None, y=h, pre=hp), dict(x=h, accf=af1, accm=am1, res=t, y=y, pre=yp)]
            t = y
        out = t
    else:
        r64 = None if res is None else R(res.double())
        out, af, am, op = _fwd_conv(t, ps[0], mods[0], r64, R)
        fwd = [dict(x=t, accf=af, accm=am, res=r64, y=out, pre=op)]
    g = R(gout.double())
    grads, bwd = [None] * (6 * len(mods)), [None] * len(mods)
    g_block = g
    for i in reversed(range(len(mods))):
        fw = fwd[i]
        if case.family == "stack" and i % 2 == 1:
            g_block = g
        skip = g_block if (case.family == "stack" and i % 2 == 0) else None
        want_dx = i > 0 or need_x
        dx, gr, st = _bwd_conv(fw["x"], ps[i], mods[i], fw["accf"], fw["accm"], g, skip, R, want_dx)
        grads[6 * i: 6 * i + 6] = gr
        bwd[i] = st
        if want_dx:
            st["dx_pre"] = dx
            g = R(dx)
    dxs = [None] * len(xs)
    if need_x:
        c0 = 0
        for j, x in enumerate(xs):
            dxs[j] = g[:, c0:c0 + x.shape[1]]
            c0 += x.shape[1]
    # the exact value of every bf16 rounding: the Function's output and input gradient, and the stages inside it
    pre = {"out": [fwd[-1]["pre"]], "dx": [bwd[0]["dx_pre"]] if need_x else [],
           "conv outputs": [fw["pre"] for fw in fwd], "out_grad": [gout.double()],
           "[df | dm]": [b["df"] for b in bwd], "input gradients": [b["dx_pre"] for b in bwd if "dx_pre" in b]}
    return dict(out=out, dxs=dxs, dres=gout.double() if case.residual else None, grads=grads, fwd=fwd, bwd=bwd, pre=pre)


def autograd_ref(case, mods, xs, res, gout):
    """float64 torch autograd of the same modules: (out, dxs, dres, grads)."""
    import copy
    ms = [copy.deepcopy(m).double() for m in mods]
    for m in ms:
        # torch refuses eps = 0; 1 + 1e-300 is 1 in float64, so the folded values are the same
        m.block['norm'].eps = max(m.block['norm'].eps, 1e-300)
    xr = [x.double().requires_grad_(case.need != "no_x") for x in xs]
    rr = None if res is None else res.double().requires_grad_(True)
    params = [p for m in ms for p in (m.block['conv_f'].weight, m.block['conv_f'].bias, m.block['conv_m'].weight,
                                      m.block['conv_m'].bias, m.block['norm'].weight, m.block['norm'].bias)]
    if case.family == "stack":
        t = xr[0]
        for r in range(0, 8, 2):
            t = ms[r + 1](ms[r](t)) + t
        out = t
    else:
        out = ms[0](torch.cat(xr, 1) if len(xr) > 1 else xr[0])
        if rr is not None:
            out = out + rr
    leaves = [x for x in xr if x.requires_grad] + ([rr] if rr is not None else []) + params
    gr = torch.autograd.grad(out, leaves, gout.double())
    n = sum(x.requires_grad for x in xr)
    dxs = list(gr[:n]) if n else [None] * len(xs)
    dres = gr[n] if rr is not None else None
    return out.detach(), dxs, dres, list(gr[n + (rr is not None):])


# ---------------------------------------------------------------- the exactness precondition
def _check_sum(what, absum, u):
    """Every partial sum of terms whose absolute values add to ``absum`` (per output element) is a multiple of ``u`` below 2^24
    units; returns the worst units."""
    m = float(absum.max()) / u if absum.numel() else 0.0
    assert m < EXACT_LIMIT, f"{what}: partial sums reach {m:.4g} units of 2^{int(math.log2(u))} >= 2^24"
    return m


def precondition(case, mods, xs, res, gout):
    """Run the replay and prove every stage exact (module docstring); returns {stage: worst units}."""
    r = replay(case, mods, xs, res, gout)
    worst = {}
    chk = lambda name, absum, u: worst.__setitem__(name, max(worst.get(name, 0.0), _check_sum(f"{case.id} {name}", absum, u)))
    for i, (fw, bw, m) in enumerate(zip(r["fwd"], r["bwd"], mods)):
        p = params64(m)
        x, wf = fw["x"], p["wf"]
        ux = unit(x)
        # forward accumulators, the epilogue's fp32 f + b_f, (f + b_f) * scale + shift [+ residual]
        chk("fwd acc", _conv(x.abs(), wf.abs(), m), ux * unit(wf))
        f = fw["accf"] + p["bf"][:, None, None]
        chk("fwd f + b_f", fw["accf"].abs() + p["bf"].abs()[:, None, None], min(ux * unit(wf), unit(p["bf"])))
        ep = (f * p["scale"][:, None, None]).abs() + p["shift"].abs()[:, None, None]
        uep = min(unit(f) * unit(p["scale"]), unit(p["shift"]))
        if fw["res"] is not None:
            ep = ep + fw["res"].abs()
            uep = min(uep, unit(fw["res"]))
        chk("fwd epilogue", ep, uep)
        assert bool((fw["accm"] == 0).all()), f"{case.id} conv {i}: the gate is not pinned (m != 0)"
        assert not m.elu or bool((bw["f"] > 0).all()), f"{case.id} conv {i}: an ELU conv with f + b_f <= 0"
        # backward: bf16(f) + b_f, dg = dy * scale, the sums over pixels, the weight and input gradients
        ug, udf = unit(bw["gy"]), unit(bw["dfr"])
        chk("bwd f + b_f", rnd(fw["accf"]).abs() + p["bf"].abs()[:, None, None], min(unit(rnd(fw["accf"])), unit(p["bf"])))
        chk("bwd dg", (bw["gy"] * p["scale"][:, None, None]).abs(), ug * unit(p["scale"]))
        pad = (m.k - 1) // 2
        if case.need != "frozen":           # a frozen Function returns no parameter gradient
            chk("dbias_f", bw["df"].abs().sum((0, 2, 3)), unit(bw["df"]))
            gm = bw["g"] - p["mean"][:, None, None]
            chk("g - mean", bw["g"].abs() + p["mean"].abs()[:, None, None], min(unit(bw["g"]), unit(p["mean"])))
            chk("dgamma", (bw["gy"].abs() * gm.abs()).sum((0, 2, 3)), ug * unit(gm))
            chk("dbeta", bw["gy"].abs().sum((0, 2, 3)), ug)
            chk("dW", torch.nn.grad.conv2d_weight(x.abs(), tuple(wf.shape), bw["dfr"].abs(), stride=m.stride, padding=pad),
                ux * udf)
        if i > 0 or case.need != "no_x":
            ds = torch.nn.grad.conv2d_input(tuple(x.shape), wf.abs(), bw["dfr"].abs(), stride=m.stride, padding=pad)
            ud = udf * unit(wf)
            if bw["skip"] is not None:
                ds, ud = ds + bw["skip"].abs(), min(ud, unit(bw["skip"]))
            chk("dx", ds, ud)
    return worst


# ---------------------------------------------------------------- coverage
def nonrep_shares(r):
    """{rounding point: share of its exact values that bf16 cannot hold}: what the round-to-nearest checks test."""
    return {k: U.bf16_nonrepresentable_fraction(torch.cat([t.flatten() for t in v])) for k, v in r["pre"].items() if v}


def filter_coverage(mods):
    """Per module: (taps with a nonzero f-filter, 8-channel input blocks with one, 8-channel output blocks with one)."""
    out = []
    for m in mods:
        w = m.block['conv_f'].weight.detach()
        nz = w != 0
        cout, cin = w.shape[:2]
        taps = int(nz.any(0).any(0).sum())
        ib = int(sum(bool(nz[:, b:b + 8].any()) for b in range(0, cin, 8)))
        ob = int(sum(bool(nz[b:b + 8].any()) for b in range(0, cout, 8)))
        out.append((taps, ib, -(-cin // 8), ob, -(-cout // 8)))
    return out


# ---------------------------------------------------------------- bounded tier
# single and multi-source convs with unpinned gates, ELU's negative branch and every BatchNorm mode, held to per-element bounds.
# Integer inputs and dyadic filters keep the RAW [f | m] recompute exact, so the gate backward sees known bf16 operands and
# bwd_exact_util.gate_ref bounds [df | dm] per element (REL_BF16 |want| + TAU T).  The statistics are re-anchored at the
# Function's own (mean, inv_std, scale, shift read from its FoldedConv; bn_fwd_exact pins them per element).  sum dy is exact
# (integer output gradients); sum dy * xhat, which the kernels form in fp32 (bn_backward_reduce), carries gate_ref's sum bound
# TAU_S T_xh into k1 and so into every [df | dm] element: E_k1 = |[df | dm] at s1 + E_s1 - [df | dm] at s1| (linear in s1).
# From there the bounds propagate linearly:
#   dbias_f / dbias_m   TAU_S T_sum + sum over pixels of E_k1 (the kernel sums its unrounded fp32 df / dm)
#   dW                  the |x|-correlation of the [df | dm] bound, plus fp32 accumulation: P 2^-24 times the |x|-correlation of
#                       |[df | dm]| + bound (P products per weight element)
#   dx                  the |w|-convolution of the [df | dm] bound plus the accumulation term, then bf16's half ulp of the result
#   dgamma              TAU_S T (eval: T_dgamma; batch: sum T_xh; per item: sum over items of T_xh, plus the items' fp32 adds)
#   output              bf16(fl(A sigmoid * scale + shift) + residual), or in train mode bn_apply of the bf16 g: REL_BF16 |y| +
#                       |scale| (REL_BF16 |g| + (TAU_FAST + EPS32) |A|) + 2 EPS32 (|g scale| + |shift| + |residual|)
# test_train_fn_exact_host.py shows each bound is at most a quarter of what a dropped / doubled / neighbouring pixel, a
# neighbouring item's statistics or a one-ulp change of one output-gradient element moves in some element.
BOUNDED_MODES = ("eval", "batch", "items")
BOUNDED_CASES = SINGLE_CASES + MULTI_CASES
U24 = 2.0 ** -24
FLT_MIN = 2.0 ** -126
DEFECT_MARGIN = 4.0


def bounded_operands(case, seed=0):
    """(module, inputs, residual, output gradient) of a bounded-tier case: inputs integers in [-4, 4], filters integers times 2^-s
    (|f|, |m| of order 2 before bias), bias_m per channel from the gate's hard regions (0, +-10, +-30, +-100 or random), bias_f
    a third of channels well negative (ELU's negative branch and A + 1 cancelling), output gradient integers in [-64, 64]."""
    gen = torch.Generator().manual_seed(zlib.crc32(f"bounded/{case.id}/{seed}".encode()))
    m = make_mods(case)[0]
    xs = [U.int_tensor((case.B, c, case.H, case.W), 4, gen, 0.2) for c in case.srcs]
    res = U.int_tensor((case.B, case.cout, case.H, case.W), 64, gen, 0.2) if case.residual else None
    x = torch.cat(xs, 1).double()
    cout, k = case.cout, case.k
    wi = [U.int_tensor((cout, case.cin, k, k), 16, gen, 0.3) for _ in range(2)]
    spread = max(float(F.conv2d(x, w.double(), stride=case.stride, padding=case.pad).std()) for w in wi)
    s = max(0, round(math.log2(max(spread, 1.0) / 2)))
    pick = lambda vals: torch.tensor(vals)[torch.randint(0, len(vals), (cout,), generator=gen)]
    bm = torch.where(torch.rand(cout, generator=gen) < 0.6, pick([0.0, 10.0, -10.0, 30.0, -30.0, 100.0, -100.0]),
                     torch.randn(cout, generator=gen) * 2)
    bf = torch.where(torch.rand(cout, generator=gen) < 0.35, pick([-3.0, -7.0, -20.0]), torch.randn(cout, generator=gen))
    if not bool((bm.abs() >= 10).any()):
        bm[0] = 30.0                        # a conv with few channels (the RGB output) still gets a saturated gate
    with torch.no_grad():
        b = m.block
        b['conv_f'].weight.copy_(wi[0] * 2.0 ** -s)
        b['conv_m'].weight.copy_(wi[1] * 2.0 ** -s)
        b['conv_f'].bias.copy_(bf)
        b['conv_m'].bias.copy_(bm)
        n = b['norm']
        n.weight.copy_(torch.rand(cout, generator=gen) + 0.5)
        n.bias.copy_(torch.randn(cout, generator=gen) * 0.5)
        n.running_mean.copy_(torch.randn(cout, generator=gen) * 0.3)
        n.running_var.copy_(torch.rand(cout, generator=gen) + 0.5)
    gout = U.int_tensor((case.B, cout) + _out_hw(case), 64, gen, 0.2)
    return [m], xs, res, gout


def _gated(case, m, xs):
    """float64 (x, accf, accm, A, g) of the bounded-tier conv; the accumulators are exact (dyadic filters, integer inputs)."""
    x = rnd(torch.cat(xs, 1).double())
    p = params64(m)
    accf, accm = _conv(x, p["wf"], m), _conv(x, p["wm"], m)
    f = accf + p["bf"][:, None, None]
    A = F.elu(f) if m.elu else f
    return x, accf, accm, A, A * torch.sigmoid(accm + p["bm"][:, None, None])


def host_stats(case, mods, xs, mode):
    """float64 statistics [items, C] a call would use (eval: the fold of the running statistics; batch / items: biased mean
    and variance of g over the call or each item), as a FoldedConv holds them: mean, inv, scale, shift."""
    m = mods[0]
    p = params64(m)
    if mode == "eval":
        return {k: p[k][None] for k in ("mean", "inv", "scale", "shift")}
    g = _gated(case, m, xs)[4]
    dims = (2, 3) if mode == "items" else (0, 2, 3)
    mean = g.mean(dims)
    var = g.var(dims, unbiased=False)
    mean, var = (mean, var) if mode == "items" else (mean[None], var[None])
    inv = 1.0 / torch.sqrt(var + m.block['norm'].eps)
    scale = p["gamma"][None] * inv
    return dict(mean=mean, inv=inv, scale=scale, shift=p["beta"][None] - mean * scale)


def bounded_ref(case, mods, xs, res, gout, mode, stats):
    """{output name: (want float64, bound)} of a bounded-tier call with the statistics ``stats`` ([items, C] float64 mean,
    inv, scale, shift; items = 1 except per item), plus 'dfm' / 'B_dfm' (concat order, NCHW) for the defect checks.
    dbeta's bound is 0: it is exact."""
    m = mods[0]
    p = params64(m)
    x, accf, accm, A, g64 = _gated(case, m, xs)
    B, C = case.B, case.cout
    items = B if mode == "items" else 1
    c4 = lambda t: t.reshape(items, C)[(torch.arange(B) * items // B)][:, :, None, None]
    sc, sh = c4(stats["scale"]), c4(stats["shift"])
    r64 = None if res is None else rnd(res.double())
    y64 = g64 * sc + sh + (0 if r64 is None else r64)
    tau_a = (X.TAU_FAST + X.EPS32) * A.abs()
    By = X.REL["bf16"] * y64.abs() + sc.abs() * (tau_a + (X.REL["bf16"] * g64.abs() if mode != "eval" else 0)) + \
        2 * X.EPS32 * ((g64 * sc).abs() + sh.abs() + (0 if r64 is None else r64.abs()))
    out = {"out": (y64, By)}

    gy = rnd(gout.double())
    P = gy.shape[2] * gy.shape[3] * (1 if mode == "items" else B)
    kind = "eval" if mode == "eval" else mode
    st = None
    if mode != "eval":
        st = dict(mean=stats["mean"], inv=stats["inv"], scale=stats["scale"])
        per = (lambda t: t.reshape(B, -1, C).sum(1)) if mode == "items" else (lambda t: t.sum(0, keepdim=True))
        st["s0"] = per(_nhwc_rows(gy))
        st["s1"] = torch.zeros_like(st["s0"])
        ref0 = _gate(rnd(accf), rnd(accm), gy, p, m.elu, kind, items, st)[0]
        sum_xh, T_xh = (ref0["sum_xh"], ref0["T_xh"]) if mode == "items" else (ref0["sum_xh"].sum(0, keepdim=True),
                                                                              ref0["T_xh"].sum(0, keepdim=True))
        st["s1"] = sum_xh
    ref, df, dm = _gate(rnd(accf), rnd(accm), gy, p, m.elu, kind, items, st)
    Tn = lambda t: _nchw(t, gy)
    T = Tn(ref["T_dfm"][:, :C])
    if mode != "eval":
        st2 = dict(st, s1=st["s1"] + U.TAU_S * T_xh)
        _, df2, dm2 = _gate(rnd(accf), rnd(accm), gy, p, m.elu, kind, items, st2)
        Ek_f, Ek_m = (df2 - df).abs(), (dm2 - dm).abs()
    else:
        Ek_f = Ek_m = torch.zeros_like(df)
    Bf = U.REL_BF16 * df.abs() + U.TAU * T + Ek_f
    Bm = U.REL_BF16 * dm.abs() + U.TAU * T + Ek_m
    T_sum = ref["T_sum"]
    # fp32 underflow: the kernels' sigmoid is exactly 0 below m = -88.7 and flushes subnormals, an absolute error of a few
    # FLT_MIN in g per pixel, and each sum may lose a subnormal per term
    tiny = P * B * FLT_MIN
    tiny_g = 16 * FLT_MIN * (gy.abs() * (1 + A.abs()) * c4(stats["inv"]).abs()).sum((0, 2, 3)) + tiny
    out["dbias_f"] = (ref["sum_df"], U.TAU_S * T_sum + Ek_f.sum((0, 2, 3)) + tiny)
    out["dbias_m"] = (ref["sum_dm"], U.TAU_S * T_sum + Ek_m.sum((0, 2, 3)) + tiny)
    if mode == "eval":
        out["dgamma"] = (ref["dgamma"], U.TAU_S * ref["T_dgamma"] + tiny_g)
    else:
        dg_want = ref["sum_xh"].sum(0)
        out["dgamma"] = (dg_want, U.TAU_S * ref["T_xh"].sum(0) + (items - 1) * U24 * 2 * (ref["sum_xh"].abs().sum(0) +
                                                                                          U.TAU_S * ref["T_xh"].sum(0)) + tiny_g)
    out["dbeta"] = (ref["dbeta"], torch.zeros(C, dtype=torch.float64))
    pad, ws = case.pad, tuple(p["wf"].shape)
    wg = lambda d, xx: torch.nn.grad.conv2d_weight(xx, ws, d, stride=case.stride, padding=pad)
    for name, d, Bd in (("dwf", df, Bf), ("dwm", dm, Bm)):
        out[name] = (wg(d, x), wg(Bd, x.abs()) + P * U24 * wg(d.abs() + Bd, x.abs()))
    wf, wm = p["wf"], p["wm"]
    dxin = lambda w, d: torch.nn.grad.conv2d_input(tuple(x.shape), w, d, stride=case.stride, padding=pad)
    dx64 = dxin(wf, df) + dxin(wm, dm)
    nterm = 2 * C * case.k * case.k
    prop = dxin(wf.abs(), Bf) + dxin(wm.abs(), Bm) + nterm * U24 * (dxin(wf.abs(), df.abs() + Bf) + dxin(wm.abs(), dm.abs() + Bm))
    Bdx = U.REL_BF16 * dx64.abs() + (1 + U.REL_BF16) * prop
    c0 = 0
    for j, xx in enumerate(xs):
        out[f"dx{j}"] = (dx64[:, c0:c0 + xx.shape[1]], Bdx[:, c0:c0 + xx.shape[1]])
        c0 += xx.shape[1]
    out["_dfm"] = (torch.cat([df, dm], 1), torch.cat([Bf, Bm], 1))
    out["_x"] = (x, None)
    return out


def defect_ratios(case, mods, xs, res, gout, mode):
    """{defect: the largest change / bound it causes over the outputs} for the host statistics: the pixel of item 0 with the
    largest [df | dm] dropped (or, the same change, doubled) from the weight gradient, and replaced by its neighbour in the input
    and weight gradients; item 0 given item 1's statistics (per item, B >= 2); the output-gradient element with the largest df
    moved by one bf16 ulp (dbeta, which would see it exactly, left out)."""
    stats = host_stats(case, mods, xs, mode)
    r = bounded_ref(case, mods, xs, res, gout, mode, stats)
    dfm, _ = r["_dfm"]
    x = r["_x"][0]
    m = mods[0]
    p = params64(m)
    C, pad, ws = case.cout, case.pad, tuple(p["wf"].shape)
    ratio = lambda ch, name: float((ch.abs() / r[name][1].clamp(min=1e-300)).max())
    best = lambda chs: max(ratio(ch, n) for n, ch in chs)
    res_ = {}
    mag = dfm[0].abs().sum(0)
    h, w = divmod(int(torch.argmax(mag)), mag.shape[1])
    one = torch.zeros_like(dfm)
    one[0, :, h, w] = dfm[0, :, h, w]
    dW = torch.nn.grad.conv2d_weight(x, (2 * C,) + ws[1:], one, stride=case.stride, padding=pad)
    res_["dropped / doubled pixel"] = best([("dwf", dW[:C]), ("dwm", dW[C:])])
    Ho, Wo = mag.shape
    h2, w2 = (h, w + 1 if w + 1 < Wo else w - 1) if Wo > 1 else (h + 1 if h + 1 < Ho else h - 1, w)
    if 0 <= h2 < Ho and 0 <= w2 < Wo:
        nb = torch.zeros_like(dfm)
        nb[0, :, h, w] = dfm[0, :, h2, w2] - dfm[0, :, h, w]
        wcat = torch.cat([p["wf"], p["wm"]], 0)
        ddx = torch.nn.grad.conv2d_input(tuple(x.shape), wcat, nb, stride=case.stride, padding=pad)
        chs, c0 = [], 0
        for j, xx in enumerate(xs):
            chs.append((f"dx{j}", ddx[:, c0:c0 + xx.shape[1]]))
            c0 += xx.shape[1]
        dWn = torch.nn.grad.conv2d_weight(x, (2 * C,) + ws[1:], nb, stride=case.stride, padding=pad)
        res_["neighbouring pixel"] = max(best(chs), best([("dwf", dWn[:C]), ("dwm", dWn[C:])]))
    if mode == "items" and case.B >= 2:
        st2 = {k: v.clone() for k, v in stats.items()}
        for k in st2:
            st2[k][0] = stats[k][1]
        r2 = bounded_ref(case, mods, xs, res, gout, mode, st2)
        res_["neighbouring item's statistics"] = best([(n, r2[n][0] - r[n][0]) for n in ("dbias_f", "dbias_m", "dwf", "dwm")])
    # the output-gradient element whose f gradient is largest
    df = dfm[:, :C] * (gout != 0)
    g2 = gout.clone()
    ix = int(torch.argmax(df.abs()))
    v = g2.view(-1)[ix]
    ulp = 2.0 ** (math.floor(math.log2(abs(float(v)))) - 7)
    g2.view(-1)[ix] = v + ulp
    r3 = bounded_ref(case, mods, xs, res, g2, mode, stats)
    res_["one-ulp output gradient"] = best([(n, r3[n][0] - r[n][0]) for n in ("dbias_f", "dwf", "dx0")])
    return res_
