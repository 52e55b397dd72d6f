"""float64 reference of the similarity and contrastive-loss kernels (csrc/loss.cu, csrc/loss_fused.cu), the bounds their
arithmetic allows, and the seeded inputs of their tests (test_loss_kernels_gpu.py; test_loss_kernels_host.py shows on
the CPU that the bounds catch deliberate faults).  Needs no GPU: every function works on the device its inputs are on.

The reference takes the fp32 values the kernels read and computes in float64:
  an = a / max(|a|, eps), x = tn vn^T, z = x / tau (the fp32 value of 1 / tau the kernels receive),
  stats = [LSE_j z_ij | LSE_{j: m_ij} z_ij | LSE_i z_ij | LSE_{i: m_ji} z_ij]   (rows over all / positive columns, then
          columns over all rows and over mask[j, i], the un-transposed mask of the reference loss),
  loss  = -mean_i (lp_r - la_r) - mean_j (lp_c - la_c),
  dX_ij = -(g / G) / tau [m_ij e^(z - lp_r_i) - e^(z - la_r_i) + m_ji e^(z - lp_c_j) - e^(z - la_c_j)],
  d an  = dX vn, d vn = dX^T tn, da = (dan - an <an, dan>) / |a| if |a| > eps, else dan / eps.

Bounds (u = 2^-24, S = 1.25 slack, all element-wise):
  norm   |a| is a warp sum of squares: every square passes through L = ceil(C/32) + 5 additions (lane loop + 5 shuffle
         levels; the fused loader always runs 8 lane steps, L = 13), so the sum is within (L + 1) u, the sqrt halves
         that and adds u: e_n = ((L + 1) / 2 + 1) u |a|.  Each element of an adds the reciprocal and the product:
         rho = e_n / |a| + 2u relative.
  x      a sequential fmaf over C (fused kernel and sgemm alike): gamma_C sum_k |an_ik vn_jk| <= (C + 2) u (|tn| |vn|^T),
         plus both rows' normalisation error, 2 rho (|tn| |vn|^T).  On the staged `nce_*` path x is an input: no term.
  z      dz = |x error| / tau + u |z|.
  LSE    mx + log S, S = sum_k e_k, e_k = exp(z_k - mx).  With p_k = e^(z_k - LSE) each term's share of its sum:
           e_LSE = S (sum_k p_k (dz_k + n_sub u a_k + 2u ulps(a_k)) + D u + 2u |log S| + u |LSE|),   a_k = mx - z_k >= 0,
         ulps = the exp's documented ulp bound: 2 for expf, 2 + floor(1.173 a) for __expf (loss.cu calls it explicitly);
         one ulp is at most 2u relative.  D = the additions of the sum: ceil(G/32) + 5 for a warp's row or column; the
         fused column sums run over the tile's <= 32 rows, then merge ceil(G/32) tile partials, each rescaled by a second
         expf (n_sub = 2, ulps doubled, D = 32 + tiles + 1).  logf is within 1 ulp, the last addition u.
  loss   sum of the four stats' bounds / G, plus the summation, D = 4 ceil(G/256) + 11 additions over
         sum |stats| / G.
  dX     every exp term carries dz + e_stat + u |z - stat| + 2u ulps(|z - stat|) relative error; the three additions and
         the coefficient g / (G tau) add 3u of the terms' magnitude sum and 3u |dX|.
  d an   sum_j dX_ij vn_jk: the errors of dX times |vn|, plus (G + 1) u + rho of sum_j |dX_ij| |vn_jk| (a sequential fmaf
         over G in the fused kernel, the sgemm's K = G loop on the staged path).
  da     s = <an, dan>: sum_k |an_k| e_dan_k + (rho + (L + 1) u) sum_k |an_k dan_k|; the numerator dan - an s adds
         |an| e_s + rho |an s| + 2u (|dan| + |an s|) -- the projection's two parts --, the division by |a| adds
         e_n / |a| + u of |da|; below eps: e_dan / eps + u |da|.
  sgemm  `assert_sum_bound` with rel = S (K + 3) u over |alpha| (|A| |B|) + |beta C|.
  max-margin  on the dyadic test grid every hinge is exact, so the gradient is an exact multiple of g = gscale / denom:
         element ij receives A_ij atomic terms of +-g (A_ii = the active hinges of anchor i); g itself is rounded once and
         an fp32 running sum of A terms is within (A - 1) u A g, so e_dx = S (A + 1) u A g -- exactly 0 where no hinge
         is active (torch's relu'(0) = 0).  The loss: exact terms, D = 2 ceil(G^2 / (256 grid)) + 11 + grid additions
         (the last is one atomicAdd per CTA) over sum |terms| / denom.

Measured on an H100 80GB HBM3 (700 W), the element-wise checks reach 0.1-0.8 of these bounds: stats 0.10 (fused) and
0.27 (nce), nce dx 0.26, norms 0.20, rownorm da 0.77, sgemm 0.08, max-margin dx 0.20, the fused gradients 0.015-0.026.
Three bounds sit further off, by construction, and are kept as they are:
  * the loss (0.009 fused, 0.0014 nce, 0.0004 staged): it adds the 4G statistics' bounds with one sign, while their
    errors have random signs and a row's lp and la share its logits' errors, which cancel in lp - la.  The statistics
    themselves are held at their own bounds, where a fault shows first;
  * the staged gradients (0.004-0.01): they carry the nce dX bound, whose __expf term is the documented worst case,
    up to 2 + 1.173 * 40 = 48 ulps at the logits' full range of 40, where the measured error is a few ulps;
  * the fused gradients: the gamma_C and gamma_G terms are worst cases for sums whose rounding errors mostly cancel.
"""
import math

import torch

F32, F64 = torch.float32, torch.float64
U = 2.0 ** -24
SLACK = 1.25
EPS = 1e-8
EPS_F32 = float(torch.tensor(EPS, dtype=F32))          # as the kernels receive it


def f32(v):
    """The value a kernel receives for the Python float v (a C float argument)."""
    return float(torch.tensor(v, dtype=F32))


def expf_ulps(a):
    return torch.full_like(a, 2.0)


def fast_expf_ulps(a):
    return 2.0 + torch.floor(1.173 * a)


# ---------------------------------------------------------------------------------------------------------- inputs
def gaussian_embeddings(G, C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(G, C, generator=g), torch.randn(G, C, generator=g)


def training_embeddings(G, C, seed):
    """The training regime: video rows are the text rows plus noise (diagonal cosines about 0.9, logits up to 18-20),
    clip 1 duplicates clip 0 (exact ties), and, where G allows, an all-zero row and a row of norm 1e-9 (below eps) on
    each side.  Returns (text, video, planted) with planted = the rows to copy tags for: [(dst, src)]."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(G, C, generator=g)
    v = t + 0.48 * torch.randn(G, C, generator=g)
    dup = []
    if G >= 4:
        t[1], v[1] = t[0], v[0]
        dup.append((1, 0))
    if G >= 8:
        t[G - 2] = 0.0
        v[G - 3] = 0.0
        t[G - 4] *= 1e-9 / t[G - 4].norm()
        v[G - 5] *= 1e-9 / v[G - 5].norm()
    elif G >= 3:
        t[G - 1] = 0.0
        v[G - 2] *= 1e-9 / v[G - 2].norm()
    return t, v, dup


def tags(G, n_verb, n_noun, seed, dup=()):
    from egovlp_b200.synthetic import synthetic_tags
    verb, noun = synthetic_tags(G, seed=seed, n_verb=n_verb, n_noun=n_noun)
    for d, s in dup:
        verb[d], noun[d] = verb[s], noun[s]
    return verb, noun


def pack_bits(t):
    """Host packing of a multi-hot [G, n] matrix: int32 [G, ceil(n/32)], bit j of word w = (t[:, 32 w + j] != 0)."""
    G, n = t.shape
    W = (n + 31) // 32
    nz = torch.zeros(G, W * 32, dtype=torch.int64)
    nz[:, :n] = (t.cpu() != 0).long()
    words = (nz.view(G, W, 32) << torch.arange(32)).sum(-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def positives(verb, noun, mode):
    """bool [G, G]: the diagonal OR (mode 1: a shared verb AND a shared noun; 2: a shared noun; 3: a shared verb)."""
    G = (verb if verb is not None else noun).shape[0]
    eye = torch.eye(G, dtype=torch.bool, device=(verb if verb is not None else noun).device)
    if mode == 0:
        return eye
    share = lambda a: (a.double() != 0).double() @ (a.double() != 0).double().T > 0
    sv = share(verb) if mode in (1, 3) else None
    sn = share(noun) if mode in (1, 2) else None
    return eye | (sv & sn if mode == 1 else sn if mode == 2 else sv)


def mask_from_sims_ref(sv, sn, mode, G):
    """(sv sn + I) > 0 per mode, in float64 (equal to fp32 on the tests' inputs, whose products are exact)."""
    eye = torch.eye(G, dtype=F64)
    m = {0: lambda: eye, 1: lambda: sv.double() * sn.double() + eye, 2: lambda: sn.double() + eye,
         3: lambda: sv.double() + eye}[mode]()
    return m > 0


def signed_sims(G, seed):
    """Non-symmetric signed 'similarity' matrices on a dyadic grid ({-1, -0.5, 0, 0.5, 1}, products exact in fp32),
    with zeros on part of the diagonal."""
    g = torch.Generator().manual_seed(seed)
    sv = (torch.randint(-2, 3, (G, G), generator=g) * 0.5).float()
    sn = (torch.randint(-2, 3, (G, G), generator=g) * 0.5).float()
    return sv, sn


# ---------------------------------------------------------------------------------------------------------- test cases
def fused_case(G, C, mode, n_verb, n_noun, seed, regime):
    """Inputs of one fused / staged EgoNCE case: text, video [G, C], verb [G, n_verb], noun [G, n_noun] (CPU fp32), the
    positives mask and the temperature."""
    if regime == "train":
        t, v, dup = training_embeddings(G, C, seed)
    else:
        (t, v), dup = gaussian_embeddings(G, C, seed), ()
    verb, noun = tags(G, n_verb, n_noun, seed, dup)
    temp = 0.05 if seed % 2 == 0 else 0.07
    return t, v, verb, noun, positives(verb, noun, mode), temp


def nce_case(G, seed):
    """A similarity matrix of the training regime (fp32, cosines), a non-symmetric positives mask (the tag mask with
    some off-diagonal entries removed on one side only) and a row (and column) whose only positive is the diagonal."""
    t, v, verb, noun, mask, temp = fused_case(G, 64, 1, 118, 582, seed, "train")
    tn, _ = normalise(t)
    vn, _ = normalise(v)
    x = (tn @ vn.T).float()
    g = torch.Generator().manual_seed(seed + 1)
    mask = mask | (torch.rand(G, G, generator=g) < 0.05)
    mask = mask & ~(torch.rand(G, G, generator=g) < 0.3).triu(1)
    mask.fill_diagonal_(True)
    mask[G // 2] = False
    mask[G // 2, G // 2] = True
    return x, mask, temp


def maxmargin_case(G, seed, adaptive):
    """x on the 2^-10 grid in [-1, 1] with the diagonal raised a little, some entries equal to diag - margin (hinges
    exactly at 0); the adaptive weight on {0, 0.5, 1, 1.5} (margin 0.25)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-1024, 1025, (G, G), generator=g).float() / 1024
    x.diagonal().copy_((torch.randint(256, 1025, (G,), generator=g).float()) / 1024)
    d = x.diagonal().clone()
    at = torch.rand(G, G, generator=g) < 0.1
    x = torch.where(at, (d[:, None] - 0.25).expand(G, G), x)
    x.diagonal().copy_(d)
    w = (torch.randint(0, 4, (G,), generator=g).float() * 0.5) if adaptive else None
    return x, w


# ---------------------------------------------------------------------------------------------------------- reference
def norm_rel(C, fused):
    L = (8 if fused else math.ceil(C / 32)) + 5
    return ((L + 1) / 2 + 1) * U


def normalise(a, eps=EPS_F32):
    a = a.to(F64)
    n = a.norm(dim=1)
    return a / n.clamp_min(eps)[:, None], n


def lse_with_bound(z, keep, mx, dz, ulps, depth, n_sub=1, exp_mult=1):
    """LSE over the last dim of z restricted to `keep`, and its bound (see the module docstring)."""
    zk = z.masked_fill(~keep, -math.inf)
    lse = torch.logsumexp(zk, -1)
    p = torch.exp(zk - lse[..., None])
    a = (mx[..., None] - z).clamp_min(0)
    e_k = dz + n_sub * U * a + exp_mult * 2 * U * ulps(a)
    err = SLACK * ((p * e_k).sum(-1) + depth * U + 2 * U * (lse - mx).abs() + U * lse.abs())
    return lse, err


def nce_reference(x, mask, inv_temp, gscale=1.0, dz=None, path="nce", col_mask=None):
    """EgoNCE on a similarity matrix x [G, G] (fp32 values) with a bool positives mask: stats [4G], loss and dX with
    their bounds.  `path` picks the LSE arithmetic: "nce" (loss.cu, __expf) or "fused" (loss_fused.cu, expf, column
    partials merged across tiles).  `dz`: the logits' error (default: the product's rounding, x being an input).
    `col_mask` overrides mask for the column sums (to model faults)."""
    x = x.to(F64)
    G = x.shape[0]
    z = x * inv_temp
    dz = U * z.abs() if dz is None else dz
    cm = mask if col_mask is None else col_mask
    allk = torch.ones_like(mask)
    warp_depth = math.ceil(G / 32) + 5
    ulps = fast_expf_ulps if path == "nce" else expf_ulps
    row = dict(ulps=ulps, depth=warp_depth)
    col = row if path == "nce" else dict(ulps=ulps, depth=min(32, G) + math.ceil(G / 32) + 1, n_sub=2, exp_mult=2)
    mr, mc = z.max(1).values, z.max(0).values
    la_r, e1 = lse_with_bound(z, allk, mr, dz, **row)
    lp_r, e2 = lse_with_bound(z, mask, mr, dz, **row)
    la_c, e3 = lse_with_bound(z.T, allk, mc, dz.T, **col)
    lp_c, e4 = lse_with_bound(z.T, cm, mc, dz.T, **col)
    stats, stats_err = torch.cat([la_r, lp_r, la_c, lp_c]), torch.cat([e1, e2, e3, e4])
    loss = -((lp_r - la_r).sum() + (lp_c - la_c).sum()) / G
    loss_err = stats_err.sum() / G + SLACK * (4 * math.ceil(G / 256) + 11) * U * stats.abs().sum() / G
    # backward
    m, mt = mask.to(F64), cm.T.to(F64)
    coef = gscale * inv_temp / G
    terms = [(m, lp_r[:, None], e2[:, None]), (-1.0, la_r[:, None], e1[:, None]),
             (mt, lp_c[None, :], e4[None, :]), (-1.0, la_c[None, :], e3[None, :])]
    t = torch.zeros_like(z)
    mag = torch.zeros_like(z)
    err = torch.zeros_like(z)
    for w, s, es in terms:
        e = torch.exp(z - s)
        arg = (z - s).abs()
        t = t + w * e
        mag = mag + abs(w) * e if isinstance(w, float) else mag + w * e
        err = err + (w.abs() if torch.is_tensor(w) else 1.0) * e * (dz + es + U * arg + 2 * U * ulps(arg))
    dx = -coef * t
    dx_err = SLACK * coef * (err + 3 * U * mag) + SLACK * 3 * U * dx.abs()
    return {"z": z, "stats": stats, "stats_err": stats_err, "loss": loss, "loss_err": loss_err, "dx": dx,
            "dx_err": dx_err}


def rownorm_bwd_reference(dan, an, n, eps, C, dan_err=None, rho=0.0, n_rel=0.0, fused=False):
    """da = (dan - an <an, dan>) / |a| above eps, dan / eps at or below, and its bound.  dan_err / rho / n_rel: the
    errors the inputs carry (none when the kernel is handed exact fp32 values)."""
    dan, an, n = dan.to(F64), an.to(F64), n.to(F64)
    dan_err = torch.zeros_like(dan) if dan_err is None else dan_err
    L = (8 if fused else math.ceil(C / 32)) + 5
    prod = (an * dan).abs()
    s = (an * dan).sum(1)
    e_s = (an.abs() * dan_err).sum(1) + (rho + (L + 1) * U) * prod.sum(1)
    proj = (an * s[:, None]).abs()
    num = dan - an * s[:, None]
    e_num = dan_err + an.abs() * e_s[:, None] + rho * proj + 2 * U * (dan.abs() + proj)
    big = (n > eps)[:, None]
    da = torch.where(big, num / n.clamp_min(eps)[:, None], dan / eps)
    e_da = torch.where(big, e_num / n.clamp_min(eps)[:, None] + (n_rel + U) * da.abs(), dan_err / eps + U * da.abs())
    return da, SLACK * e_da


def egonce_reference(text, video, mask, inv_temp, path, gscale=1.0, eps=EPS_F32, col_mask=None, norm_fn=None):
    """sim_matrix + EgoNCE from the embeddings (fp32 values): the similarities, stats, loss and d text / d video, each
    with its bound.  path: "fused" (loss_fused.cu) or "staged" (rownorm + sgemm + nce_*)."""
    G, C = text.shape
    fused = path == "fused"
    tn, nt = (norm_fn or normalise)(text, eps)
    vn, nv = (norm_fn or normalise)(video, eps)
    x = tn @ vn.T
    xt = tn.abs() @ vn.abs().T
    nrel = norm_rel(C, fused)
    rho = nrel + 2 * U
    x_err = ((C + 2) * U + 2 * rho) * xt
    r = nce_reference(x, mask, inv_temp, gscale, dz=inv_temp * x_err + U * (x * inv_temp).abs(),
                      path="fused" if fused else "nce", col_mask=col_mask)
    dx, dx_err = r["dx"], r["dx_err"]
    out = dict(r, x=x, x_err=SLACK * x_err, tn=tn, vn=vn, norm_text=nt, norm_video=nv,
               norm_text_err=SLACK * nrel * nt, norm_video_err=SLACK * nrel * nv)
    for side, a, na, b, d, de in (("text", tn, nt, vn, dx, dx_err), ("video", vn, nv, tn, dx.T, dx_err.T)):
        dan = d @ b
        dan_err = de @ b.abs() + ((G + 1) * U + rho) * (d.abs() @ b.abs())
        da, e = rownorm_bwd_reference(dan, a, na, eps, C, dan_err=SLACK * dan_err, rho=rho, n_rel=nrel, fused=fused)
        out["d_" + side], out["d_" + side + "_err"] = da, e
    return out


def maxmargin_reference(x, margin, fix_norm, weight=None, gscale=1.0):
    """MaxMarginRankingLoss (AdaptiveMaxMarginRankingLoss with `weight`): loss and dx, each with its bound."""
    x = x.to(F64)
    G = x.shape[0]
    d = x.diagonal()[:, None]
    m = (torch.full((G,), f32(margin), dtype=F64, device=x.device) if weight is None
         else f32(margin) * weight.to(F64))[:, None]
    h1, h2 = m - (d - x), m - (d - x.T)
    off = ~torch.eye(G, dtype=torch.bool, device=x.device) if fix_norm else torch.ones_like(x, dtype=torch.bool)
    a1, a2 = ((h1 > 0) & off).to(F64), ((h2 > 0) & off).to(F64)
    denom = 2.0 * G * (G - 1) if fix_norm else 2.0 * G * G
    terms = (h1.clamp_min(0) * off + h2.clamp_min(0) * off)
    loss = terms.sum() / denom
    g = gscale / denom
    A = a1 + a2.T + torch.diag(a1.sum(1) + a2.sum(1))              # atomic terms per element, in units of g
    dx = g * (a1 + a2.T) - g * torch.diag(a1.sum(1) + a2.sum(1))
    n = G * G
    grid = min(1024, (n + 255) // 256)
    depth = 2 * math.ceil(n / (256 * grid)) + 11 + grid
    return {"loss": loss, "loss_err": SLACK * depth * U * terms.sum() / denom + 1e-30, "dx": dx,
            "dx_err": SLACK * (A + 1) * U * A * g, "active": A}


def sgemm_reference(a, b, alpha, beta, c0):
    """alpha a @ b^T + beta c0 ([M, K] x [N, K]) and the magnitude sum of its terms."""
    a, b = a.to(F64), b.to(F64)
    out = alpha * (a @ b.T)
    mag = abs(alpha) * (a.abs() @ b.abs().T)
    if beta != 0.0:
        out = out + beta * c0.to(F64)
        mag = mag + abs(beta) * c0.to(F64).abs()
    return out, mag
