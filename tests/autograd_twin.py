"""A float64 autograd restatement of the differentiable half of Renderer::Render plus the trainer's loss.

Test infrastructure.  It runs no project kernel and does not use the CPU oracle: plain torch in float64, on the CPU or on CUDA.
Its gradients come from autograd, so they do not share the hand derivation that both the CUDA backward
(f2nerf_b200/csrc/*.cu) and the CPU oracle (oracle/f2_oracle.c) are written from.  Only three reference operators get their
backward written out, because their backward is not the derivative of their forward (TruncExp, GradientScaling, WeightVar).

The non-differentiable part of a step comes in as data: the kept samples (pts, t, dt, volume ids) with their ray bounds, the
background, the per-ray camera index, the TV-loss edge points with their volume ids, the SH4 encoding of the directions and
the per-level scales of the hash encode (the device's exp2f values).  The leaves are the table [pool, 2], the two MLP parameter
vectors in tiny-cuda-nn's [out][in] layout and the appearance embedding.

``dev`` pins the forward to the values a run under test computed: a stage's output ``x`` becomes ``x + (dev - x).detach()``
(after checking it lies within one fp16 ulp of ``dev``), so the forward is bit for bit the run's own and the gradient still
flows through ``x``.  What is left between a backward under test and the twin is the fp16 rounding of the rows that backward
writes (loss-scaled dL/dout, the hidden-layer gradients, dL/dfeat).

``broken`` names deliberate mistakes (BROKEN); the tests use them to show their bars catch an error of that size.
"""
import torch

F64 = torch.float64
N_LEVELS = 16
BROKEN = ("gs_linear", "truncexp_noclamp", "emb_15ch", "weightvar_centered", "disp_no_eps")


# ---------------------------------------------------------------------------------------------------------------- pinning
def fp16_ulp(v):
    """One fp16 ulp at |v| (2^-24 in the subnormal range)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


class Pins:
    """Records, per pinned stage, the largest distance from the run's value in fp16 ulps and how many values the twin's own
    fp16 rounding would put on a different fp16 number (``flips``)."""

    def __init__(self):
        self.stats = {}

    def pin(self, name, x, dev, scale=None, tol=1.0):
        """Checks |x - dev| <= 1 fp16 ulp, taken at |dev| or, for a sum, at ``scale`` = the sum of the magnitudes of its terms
        when that is larger: the run sums in fp32 where the twin sums in float64 (an MLP output also has its hidden layer
        rounded from a different sum), so an output that cancels may differ by a fraction of an ulp of its terms.  ``tol``: the
        ulps allowed, 1 unless the run rounds twice."""
        if dev is None:
            return x
        d = dev.to(device=x.device, dtype=F64).reshape(x.shape)
        at = d.abs() if scale is None else torch.maximum(d.abs(), scale.detach().reshape(x.shape))
        err = ((x.detach() - d).abs() / fp16_ulp(at)) if x.numel() else x.detach()
        flips = int((x.detach().half() != dev.to(x.device).reshape(x.shape).half()).sum()) if x.numel() else 0
        worst = float(err.max()) if x.numel() else 0.0
        self.stats[name] = dict(max_ulp=worst, flips=flips, n=int(x.numel()))
        assert worst <= tol + 1e-6, f"{name}: twin forward {worst:.3f} fp16 ulp away from the run's"
        return x + (d - x).detach()


def round16(x):
    """fp16 storage of a value the run does not keep (the fp16 table and parameters the forward reads, the MLP hidden layers):
    rounded forward, straight-through backward."""
    return x + (x.detach().half().to(F64) - x.detach())


# ------------------------------------------------------------------------------------------------- the three reference rules
class TruncExp(torch.autograd.Function):
    """CustomOps.cpp:9-18: exp forward; backward g * exp(clamp(x, -100, 5))."""

    @staticmethod
    def forward(ctx, x, clamp=True):
        ctx.save_for_backward(x)
        ctx.clamp = clamp
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        return g * torch.exp(x.clamp(-100., 5.) if ctx.clamp else x), None


class GradientScaling(torch.autograd.Function):
    """CustomOps.cu:68-80,127-166: identity forward; backward multiplies row i of a ray of n kept samples by
    p + (1 - p) a^2, a = (i + .5) / n."""

    @staticmethod
    def forward(ctx, x, scale):
        ctx.save_for_backward(scale)
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        scale, = ctx.saved_tensors
        return g * (scale if g.dim() == 1 else scale[:, None]), None


class WeightVar(torch.autograd.Function):
    """CustomOps.cu:12-66.  Forward: per ray, mean = sum w_i x_i / W, var = sum w_i (x_i - mean)^2 with x_i = i / 16 and
    W = 1e-6 + sum w_i.  Backward, as the reference writes it: dl/dw_j = bias_j^2 + tmp * (-x_j) / W with bias_j = x_j - mean,
    tmp = sum 2 w_i bias_i.  The exact derivative has (x_j - mean) where the reference has x_j; the twin follows the reference
    (``centered`` gives the exact derivative, a deliberate deviation).  The two differ by tmp * mean / W, and tmp is 2e-6 mean,
    so they part only on rays whose total weight is near 1e-6."""

    @staticmethod
    def forward(ctx, w, seg, centered=False):
        rid, pos, n_rays = seg["rid"], seg["pos"], seg["n_rays"]
        x = pos.to(F64) / 16.
        W = torch.zeros(n_rays, dtype=F64, device=w.device).index_add_(0, rid, w) + 1e-6
        mean = torch.zeros(n_rays, dtype=F64, device=w.device).index_add_(0, rid, w * x) / W
        bias = x - mean[rid]
        var = torch.zeros(n_rays, dtype=F64, device=w.device).index_add_(0, rid, w * bias * bias)
        tmp = torch.zeros(n_rays, dtype=F64, device=w.device).index_add_(0, rid, w * 2. * bias)
        ctx.save_for_backward(x, bias, W, tmp, rid)
        ctx.centered = centered
        return var

    @staticmethod
    def backward(ctx, g):
        x, bias, W, tmp, rid = ctx.saved_tensors
        xj = bias if ctx.centered else x
        return g[rid] * (bias * bias + tmp[rid] * -xj / W[rid]), None, None


# ---------------------------------------------------------------------------------------------------------------- pieces
def segments(bounds):
    """Per kept sample: its ray (rid), its index inside the ray (pos) and the ray's kept count (n); bounds [R, 2] packed."""
    b = bounds.to(torch.int64)
    cnt = b[:, 1] - b[:, 0]
    rid = torch.repeat_interleave(torch.arange(b.shape[0], device=b.device), cnt)
    pos = torch.arange(rid.shape[0], device=b.device) - b[rid, 0]
    return dict(rid=rid, pos=pos, n=cnt[rid], n_rays=b.shape[0])


def _mul_lo32(a, p):
    """(a * p) mod 2^32 for a, p in [0, 2^32) held in int64, without overflowing."""
    lo = a * (p & 0xFFFF)
    hi = ((a * (p >> 16)) & 0xFFFF) << 16
    return (lo + hi) & 0xFFFFFFFF


def hash_corners(pts, vol, level, hp):
    """Hash3DAnchored.cu:27-66 for one level: table rows [n, 8] and trilinear weights [n, 8] (float64).
    hp: dict(prim int64 [16 * V, 3], bias float32 [16 * V, 3], scales float32 [16], local_size)."""
    S = int(hp["local_size"])
    x = (pts.to(torch.float32) + 1.) * .5                                  # Hash3DAnchored.cpp:91
    tv = level * hp["n_volumes"] + vol.to(torch.int64)
    bias = hp["bias"][tv]
    # pt * mul + bias with one rounding to fp32 (the product of two floats is exact in float64)
    p = (x.to(F64) * float(hp["scales"][level]) + bias.to(F64)).to(torch.float32)
    fl = torch.floor(p)
    i = fl.to(F64).clamp(0., 4294967295.).to(torch.int64)                 # static_cast<unsigned>: saturating
    frac = (p - fl).to(F64)
    prim = hp["prim"][tv]
    h0 = [_mul_lo32(i[:, k], prim[:, k]) for k in range(3)]
    h1 = [_mul_lo32((i[:, k] + 1) & 0xFFFFFFFF, prim[:, k]) for k in range(3)]
    rows, ws = [], []
    for c in range(8):                                                     # corner order 000, 001, ..., 111 (x, y, z bits)
        bx, by, bz = (c >> 2) & 1, (c >> 1) & 1, c & 1
        h = (h1[0] if bx else h0[0]) ^ (h1[1] if by else h0[1]) ^ (h1[2] if bz else h0[2])
        # level l starts at HALF-element l * local_size of the [pool, 2] table: row l * S / 2 (hash.cuh:61's overlap)
        rows.append(level * (S // 2) + h % S)
        w = (frac[:, 0] if bx else 1. - frac[:, 0]) * (frac[:, 1] if by else 1. - frac[:, 1]) * (frac[:, 2] if bz else 1. - frac[:, 2])
        ws.append(w)
    return torch.stack(rows, 1), torch.stack(ws, 1)


def _encode_level(table, pts, vol, hp, level):
    rows, w = hash_corners(pts, vol, level, hp)
    return (w[:, :, None] * table[rows]).sum(1)


def hash_encode(table, pts, vol, hp, levels=range(N_LEVELS)):
    """[n, 32] float64 features (level-major, 2 channels each) of the points from the float64 table leaf.  Each level is
    recomputed in the backward (torch.utils.checkpoint), so a batch of millions of points holds one level's gather at a time."""
    from torch.utils.checkpoint import checkpoint
    out = []
    for l in levels:
        if table.requires_grad:
            out.append(checkpoint(_encode_level, table, pts, vol, hp, l, use_reentrant=False))
        else:
            out.append(_encode_level(table, pts, vol, hp, l))
    return torch.cat(out, 1)


def mlp(x, params, n_hidden_matmuls, magnitude=False):
    """tiny-cuda-nn FullyFusedMLP, width 64, ReLU, no bias: params [W0 64x32 | Wh 64x64 * nh | Wout 16x64] ([out][in]).
    ``magnitude``: also return sum_j |h_j W_ij| of the output layer."""
    W0 = params[:64 * 32].view(64, 32)
    h = round16(torch.relu(x @ W0.T))
    o = 64 * 32
    for _ in range(n_hidden_matmuls):
        h = round16(torch.relu(h @ params[o:o + 64 * 64].view(64, 64).T))
        o += 64 * 64
    Wo = params[o:o + 16 * 64].view(16, 64)
    if magnitude:
        return h @ Wo.T, h.detach().abs() @ Wo.detach().abs().T
    return h @ Wo.T


def shader_act(raw):
    """SHShader.cpp:27-28 on the first three outputs."""
    return (1. + 2e-3) * torch.sigmoid(raw[:, :3]) - 1e-3


def seg_sum(v, seg):
    return torch.zeros((seg["n_rays"],) + v.shape[1:], dtype=v.dtype, device=v.device).index_add(0, seg["rid"], v)


def gs_scale(seg, progress, linear=False):
    a = (seg["pos"].to(F64) + .5) / seg["n"].to(F64)
    return progress + (1. - progress) * (a if linear else a * a)


# ---------------------------------------------------------------------------------------------------------------- render
def render(leaves, inp, hp, dev=None, broken=(), pins=None):
    """Renderer.cpp:152-208 on the kept samples.

    leaves: dict(table [pool, 2], field [3072], shader [7168], app_emb [n_img, 16] or None), float64.
    inp: dict(pts [nk, 3], vol [nk], dt [nk], t [nk], bounds [R, 2], bg [R, 3], cam [R] or None, sh [nk, 16],
              e_pts [ne, 3], e_vol [ne], gs_progress).
    dev: dict(feat [nk + ne, 32], logit [nk], mlp_in [nk, 32], raw [nk, 16], rgb [nk, 3], edge [ne, 16]; optionally the
         composite's weights [nk], colors [R, 3], disparity [R], depth [R]) or None.
    Returns dict(colors, disparity, depth, weights, edge_feats [ne / 2, 2, 16], feat, seg)."""
    bad = set(broken)
    assert bad <= set(BROKEN), bad
    pins = Pins() if pins is None else pins
    nk = inp["pts"].shape[0]
    ne = inp["e_pts"].shape[0] if inp.get("e_pts") is not None else 0
    q_pts = torch.cat([inp["pts"], inp["e_pts"]]) if ne else inp["pts"]
    q_vol = torch.cat([inp["vol"], inp["e_vol"]]) if ne else inp["vol"]
    # the forward reads fp16 copies of the table and the parameters (Hash3DAnchored.cu:186, TCNNWP.cpp)
    table16 = round16(leaves["table"])
    feat = hash_encode(table16, q_pts, q_vol, hp)
    if dev is not None:                                   # the run sums the eight corners in fp32: 1 ulp at sum_c w_c |t_c|
        with torch.no_grad():
            mag_feat = hash_encode(table16.detach().abs(), q_pts, q_vol, hp)
        feat = pins.pin("feat", feat, dev["feat"][:nk + ne], mag_feat)
    out, mag = mlp(feat, round16(leaves["field"]), 0, magnitude=True)
    logit = pins.pin("logit", out[:nk, 0], None if dev is None else dev["logit"][:nk], mag[:nk, 0])
    edge = pins.pin("edge", out[nk:], None if dev is None else dev["edge"][:ne], mag[nk:]) if ne else out[nk:]
    seg = segments(inp["bounds"])
    # shading input (Renderer.cpp:181-187): channel 0 is the constant 1, the embedding is added to all 16 channels
    # the field output is stored in fp16 and the sum with the embedding rounded again: two roundings, hence 1.5 ulp below
    shading = torch.cat([torch.ones_like(out[:nk, :1]), round16(out[:nk, 1:16])], 1)
    mag_in = torch.cat([torch.ones_like(mag[:nk, :1]), mag[:nk, 1:16]], 1)
    if leaves.get("app_emb") is not None:
        emb = leaves["app_emb"][inp["cam"].to(torch.int64)[seg["rid"]]]
        if "emb_15ch" in bad:                                               # same value, no gradient into channel 0
            emb = torch.cat([emb[:, :1].detach(), emb[:, 1:]], 1)
        shading = shading + emb
        mag_in = mag_in + emb.detach().abs()
    sh = inp["sh"].to(F64)
    mlp_in = pins.pin("mlp_in", torch.cat([shading, sh], 1), None if dev is None else dev["mlp_in"][:nk], torch.cat([mag_in, sh.abs()], 1),
                     tol=1.5)
    raw, mag = mlp(mlp_in, round16(leaves["shader"]), 1, magnitude=True)
    raw = pins.pin("raw", raw, None if dev is None else dev["raw"][:nk], mag)
    rgb = pins.pin("rgb", shader_act(raw), None if dev is None else dev["rgb"][:nk])
    logit_in, rgb_in, raw_in = logit, rgb, raw
    # composite (Renderer.cpp:179,190-208)
    dens = TruncExp.apply(logit - 3., "truncexp_noclamp" not in bad)
    gs = float(inp.get("gs_progress", 1.0))
    if gs < 1.:
        scale = gs_scale(seg, gs, linear="gs_linear" in bad)
        dens = GradientScaling.apply(dens, scale)
        rgb = GradientScaling.apply(rgb, scale)
    tau = dens * inp["dt"].to(F64)
    # exclusive per-ray cumsum on a [rays, longest ray] layout: a running sum over the whole batch would lose a ray's optical
    # depth against the 1e13-sized ones of opaque samples before it
    n_max = int(seg["n"].max()) if tau.numel() else 0
    grid = tau.new_zeros((seg["n_rays"], n_max + 1)).index_put((seg["rid"], seg["pos"] + 1), tau)
    acc = torch.cumsum(grid, 1)[seg["rid"], seg["pos"]]
    weights = torch.exp(-acc) * (1. - torch.exp(-tau))
    last_trans = torch.exp(-seg_sum(tau, seg))
    colors = seg_sum(weights[:, None] * rgb, seg) + last_trans[:, None] * inp["bg"].to(F64)
    t = inp["t"].to(F64)
    ts = t if "disp_no_eps" in bad else t + 1e-2
    disparity = seg_sum(weights / ts, seg)
    depth = seg_sum(weights * (t + 1e-2), seg) / (1. - last_trans + 1e-4)
    if dev is not None and "colors" in dev:
        # the run's fp32 composite outputs: the loss is evaluated where the run evaluated it (the colour loss's slope changes
        # by 1e-4 for a 1e-6 change of a colour near its target, so float64 colours would move dL/dcolour by itself).  The
        # depth's 1 / (1 - last_trans + 1e-4) amplifies the fp32 rounding of last_trans on nearly transparent rays
        depth_at = depth.detach().abs() * (1. + 2. ** -9 / (1. - last_trans.detach() + 1e-4))
        # alpha = 1 - exp(-tau) in fp32 carries ~2^-22 absolute: relative 2^-22 / alpha of a weight
        alpha = (1. - torch.exp(-tau)).detach()
        weights = pins.pin("weights", weights, dev["weights"][:nk], weights.detach().abs() * (1. + 2. ** -10 / alpha.clamp_min(1e-300)))
        colors = pins.pin("colors", colors, dev["colors"])
        disparity = pins.pin("disparity", disparity, dev["disparity"])
        depth = pins.pin("depth", depth, dev["depth"], depth_at)
    return dict(colors=colors, last_trans=last_trans, disparity=disparity, depth=depth, weights=weights, edge_feats=edge.reshape(-1, 2, 16),
                feat=feat, logit=logit_in, rgb=rgb_in, raw=raw_in, edge=edge, seg=seg, pins=pins.stats)


# ---------------------------------------------------------------------------------------------------------------- loss
TERMS = ("color", "var", "disp", "tv", "depth")
TRAINER_MIX = dict(color=1.0, var=0.01, disp=0.01, tv=0.1)          # ExpRunner.cpp:116-118 past var_loss_end


def loss_terms(out, gt, broken=()):
    """ExpRunner.cpp:94-106, one term at a time (depth: a squared-depth term, for the d_depth path the trainer leaves unused)."""
    terms = dict(color=torch.sqrt((out["colors"] - gt.to(F64)) ** 2 + 1e-4).mean(),
                 var=torch.sqrt(WeightVar.apply(out["weights"], out["seg"], "weightvar_centered" in broken) + 1e-2).mean(),
                 disp=(out["disparity"] ** 2).mean(),
                 depth=(out["depth"] ** 2).mean())
    e = out["edge_feats"]
    terms["tv"] = ((e[:, 0] - e[:, 1]) ** 2).mean() if e.numel() else out["colors"].sum() * 0.
    return terms


def loss(out, gt, weights, broken=()):
    terms = loss_terms(out, gt, broken)
    return sum(float(w) * terms[k] for k, w in weights.items() if w)


def abs_table_contributions(table_shape, pts, vol, hp, d_feat, device=None):
    """Sum over every (point, level, corner) of |w * dL/dfeat| per table entry: the scale an fp32-accumulated table gradient
    entry is summed at."""
    tab = torch.zeros(table_shape, dtype=F64, device=device, requires_grad=True)
    f = hash_encode(tab, pts, vol, hp)
    g, = torch.autograd.grad((f * d_feat.abs().to(F64)).sum(), tab)
    return g
