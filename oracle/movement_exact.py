"""References of the pooling, padding, phase-shift, gather, one-hot, fill, softmax and cross-entropy kernels (elementwise.cu,
surface.cu) in their C-ABI layouts, a restatement of their launch configuration, and a priori error bounds for the two
transcendental kernels.

Layouts are those of include/pnp_b200.h: activations NHWC fp32, a phase-shift source X = [B, a, b, G*r*r] whose group g owns
channels [g*r*r, (g+1)*r*r), the phase-shifted output placed at channels [coff, coff + ntile*G) of a Ctot-channel tensor in
tf.tile's order [g0 .. g(G-1) g0 .. g(G-1) ...].

Pure data movement is written as explicit index maps (torch gathers, any device), so the references run next to the kernels at
the grid-stride cap.  Every reference takes the flag of one plausible kernel bug (first=False, col_major=True, reflect=True, ...):
tests/test_movement_exact_cpu.py checks that each bug changes the reference output on the GPU file's operands."""
from collections import namedtuple

import torch

from oracle.elementwise_exact import NUM_SMS, grid_for

CAP = NUM_SMS * 64            # grid_for's CTA cap
THREADS = 256                 # every launcher of this family runs 256-thread CTAs
U = 2.0 ** -24                # unit roundoff of fp32
FLT_MAX = 3.4028234663852886e38
CE_CLIP_LO = float(torch.tensor(1e-10, dtype=torch.float32))   # the kernels' 1e-10f
PS2_CLIPPED = float(torch.tensor(-1e15, dtype=torch.float32))  # fminf(fmaxf(NaN, -1e15f), 1e15f)


def _cdiv(a, b):
    return -(-a // b)


def gamma(k):
    """gamma_k = k u / (1 - k u): the relative error bound of k fp32 roundings (Higham, Lemma 3.1)"""
    return k * U / (1 - k * U)


# ------------------------------------------------------------------------------------------------
# launch configuration (132 SMs, 256 threads per CTA)
# ------------------------------------------------------------------------------------------------
# grid, whether grid_for's cap applied, the grid-stride iterations of the busiest thread, and whether the launch is one CTA
# that its items do not fill
Launch = namedtuple("Launch", "grid capped iters single_partial")


def grid_stride(items, per_block):
    """a grid-stride launch of grid_for(items, per_block) CTAs over `items` loop iterations"""
    g = grid_for(items, per_block)
    return Launch(g, _cdiv(items, per_block) > CAP, _cdiv(items, g * THREADS) if items > 0 else 0,
                  g == 1 and items < per_block)


def maxpool2_launch(B, H, W, C):
    """pnp_maxpool2_fwd / _bwd: the float4-wide template (V = 4, one thread per 4 channels, grid_for(total / 4, 512)) when
    C % 4 == 0, else V = 1 with grid_for(total, 1024); total = B * (H/2) * (W/2) * C -> (V, Launch)"""
    total = B * (H // 2) * (W // 2) * C
    if C % 4 == 0:
        return 4, grid_stride(total // 4, 512)
    return 1, grid_stride(total, 1024)


def avgpool2_launch(B, H, W, C):
    return grid_stride(B * (H // 2) * (W // 2) * C, 1024)


def pool_geom(H, W, n, round_up=False):
    """TF 'SAME' with ksize = stride = n: (Ho, Wo, pad_top, pad_left); round_up=True rounds the split up (a negative control)"""
    Ho, Wo = _cdiv(H, n), _cdiv(W, n)
    pt, pl = Ho * n - H, Wo * n - W
    return (Ho, Wo, _cdiv(pt, 2), _cdiv(pl, 2)) if round_up else (Ho, Wo, pt // 2, pl // 2)


def pool_launch(B, H, W, C, n, backward):
    """pnp_pool_fwd: one thread per output, pnp_pool_bwd: one per input element; 1024 items per CTA"""
    Ho, Wo, _, _ = pool_geom(H, W, n)
    return grid_stride(B * (H * W if backward else Ho * Wo) * C, 1024)


def crop_concat_launch(B, H1, W1, C1, H2, W2, C2, backward, dx1=True, dx2=True):
    """forward: one thread per output element; backward: one per element of dx1 then dx2 (a NULL output has none); 1024 per CTA"""
    if not backward:
        return grid_stride(B * H2 * W2 * (C1 + C2), 1024)
    return grid_stride((B * H1 * W1 * C1 if dx1 else 0) + (B * H2 * W2 * C2 if dx2 else 0), 1024)


def mirror_pad_launch(B, H, W, C, p, backward):
    """forward: one thread per padded output element, backward: one per dx element; 2048 per CTA"""
    return grid_stride(B * H * W * C if backward else B * (H + 2 * p) * (W + 2 * p) * C, 2048)


def phase_shift_launch(B, a, b, G, r):
    """forward: one thread per (output pixel, group), writing its ntile copies; backward: one per dX element; 2048 per CTA"""
    return grid_stride(B * a * b * G * r * r, 2048)


def channel_slice_launch(M, Cs):
    return grid_stride(M * Cs, 2048)


def pixel_launch(P):
    """pnp_logits_argmax_concat, pnp_pixel_softmax2, pnp_one_hot: one thread per pixel, 512 per CTA"""
    return grid_stride(P, 512)


FillLaunch = namedtuple("FillLaunch", "grid capped iters tail")


def fill_launch(n):
    """pnp_fill: grid_for(n / 4 + 1, 1024) CTAs store the n / 4 float4s; the first n % 4 threads of CTA 0 store the tail"""
    q = n // 4
    g = grid_for(q + 1, 1024)
    return FillLaunch(g, _cdiv(q + 1, 1024) > CAP, _cdiv(q, g * THREADS), n % 4)


CE_FLUSH = 32                 # cross_entropy_acc_kernel moves its fp32 partial into fp64 every 32 elements of a thread


def ce_acc_launch(n):
    """pnp_cross_entropy_fwd: grid_for(n, 4096); iters = elements of the busiest thread (> CE_FLUSH: several fp32 partials)"""
    return grid_stride(n, 4096)


def ce_bwd_launch(n):
    return grid_stride(n, 1024)


def disc_lines(Gs, ntiles):
    """distinct (source, group) lines of a plan: tiled copies share their source's lines"""
    return sum(Gs)


def disc_ctot(Gs, ntiles, NC):
    return sum(G * t for G, t in zip(Gs, ntiles)) + NC + 1


def disc_input_launch(B, a, b, r, order_b1, Gs, ntiles, NC):
    """pnp_disc_input_fwd's choice -> (path, Launch).  'r8': r == 8, the batch >= 2 sub-pixel order and at most 32 distinct lines;
    one CTA per 4 horizontally adjacent source pixels, B * a * ceil(b / 4) CTAs, no grid stride, a ragged last CTA per source
    row when b % 4 != 0.  Otherwise 'generic': one thread per (pixel, 4 output channels), grid_for(B * H * W * Ctot / 4, 256)."""
    Q = disc_ctot(Gs, ntiles, NC) // 4
    if r == 8 and not order_b1 and 0 < disc_lines(Gs, ntiles) <= 32:
        blocks = B * a * _cdiv(b, 4)
        return "r8", Launch(blocks, False, 1, blocks == 1 and b < 4)
    return "generic", grid_stride(B * a * r * b * r * Q, 256)


# ------------------------------------------------------------------------------------------------
# pooling
# ------------------------------------------------------------------------------------------------
def _axis_map(L, n, pad, Lo):
    """[Lo, n] input index of each window position along one axis (clamped) and whether it lies inside the map"""
    i = torch.arange(Lo)[:, None] * n - pad + torch.arange(n)[None, :]
    return i.clamp(0, L - 1), (i >= 0) & (i < L)


def pool_windows(x, n, round_up=False, col_major=False):
    """x [B, H, W, C] -> (win [B, Ho, Wo, C, n*n], valid [1, Ho, Wo, 1, n*n]) in row-major window order (col_major=True: the
    transposed order, a negative control)"""
    B, H, W, C = x.shape
    Ho, Wo, pt, pl = pool_geom(H, W, n, round_up)
    iy, vy = _axis_map(H, n, pt, Ho)
    ix, vx = _axis_map(W, n, pl, Wo)
    dev = x.device
    g = x[:, iy.reshape(-1).to(dev)][:, :, ix.reshape(-1).to(dev)].view(B, Ho, n, Wo, n, C)
    v = (vy[:, :, None, None] & vx[None, None, :, :]).to(dev)          # [Ho, n, Wo, n]
    if col_major:
        g, v = g.permute(0, 1, 3, 5, 4, 2), v.permute(0, 2, 3, 1)
    else:
        g, v = g.permute(0, 1, 3, 5, 2, 4), v.permute(0, 2, 1, 3)
    return g.reshape(B, Ho, Wo, C, n * n), v.reshape(1, Ho, Wo, 1, n * n)


def pool_max_ref(x, n, round_up=False):
    """tf.nn.max_pool 'SAME' n x n: the max over the valid elements of each window (padding never wins)"""
    win, valid = pool_windows(x, n, round_up)
    return torch.where(valid, win, torch.full_like(win, float("-inf"))).amax(-1)


def pool_avg_ref(x, n, round_up=False, full_count=False):
    """tf.nn.avg_pool 'SAME' n x n -> (y32, y64, magnitude, count): y32 = fl32(exact sum) / count in fp32 (what the kernel returns
    whenever its fp32 running sum is exact, e.g. on small integers), y64 the fp64 mean, magnitude sum|x| / count.
    full_count=True divides by n*n (a negative control)."""
    win, valid = pool_windows(x, n, round_up)
    w = torch.where(valid, win.double(), torch.zeros((), dtype=torch.float64, device=x.device))
    s = w.sum(-1)
    cnt = (valid.sum(-1).expand_as(s) if not full_count else torch.full_like(s, n * n)).double()
    return s.float() / cnt.float(), s / cnt, w.abs().sum(-1) / cnt, cnt


def _window_pos(H, W, n, round_up, dev):
    """per input pixel: its window (oy, ox) and its position k = ky * n + kx inside it"""
    _, _, pt, pl = pool_geom(H, W, n, round_up)
    yy, xx = torch.arange(H, device=dev) + pt, torch.arange(W, device=dev) + pl
    return yy // n, xx // n, (yy % n)[:, None] * n + (xx % n)[None, :]


def pool_max_bwd_ref(x, dy, n, first=True, col_major=False, round_up=False):
    """MaxPoolGrad: each window's gradient goes to its first maximal valid element in row-major order, every other element gets
    +0; a window of -inf routes to its first valid element.  first=False takes the last maximum, col_major=True scans the window
    column by column (negative controls)."""
    B, H, W, C = x.shape
    win, valid = pool_windows(x, n, round_up, col_major)
    m = torch.where(valid, win, torch.full_like(win, float("-inf"))).amax(-1, keepdim=True)
    hit = valid & (win == m)
    k = torch.arange(n * n, device=x.device)
    if first:
        sel = torch.where(hit, k, torch.full_like(k, n * n)).amin(-1)
    else:
        sel = torch.where(hit, k, torch.full_like(k, -1)).amax(-1)
    if col_major:                                           # back to the row-major position of the selected element
        sel = (sel % n) * n + sel // n
    oy, ox, pos = _window_pos(H, W, n, round_up, x.device)
    s = sel[:, oy][:, :, ox]                                # [B, H, W, C]
    g = dy[:, oy][:, :, ox]
    return torch.where(s == pos[None, :, :, None], g, torch.zeros_like(g))


def pool_avg_bwd_ref(dy, H, W, n, round_up=False, full_count=False):
    """AvgPoolGrad: dx = dy / (valid count of its window), one IEEE fp32 division"""
    Ho, Wo, pt, pl = pool_geom(H, W, n, round_up)
    _, vy = _axis_map(H, n, pt, Ho)
    _, vx = _axis_map(W, n, pl, Wo)
    cnt = (vy.sum(1)[:, None] * vx.sum(1)[None, :]).to(dy.device)
    if full_count:
        cnt = torch.full_like(cnt, n * n)
    oy, ox, _ = _window_pos(H, W, n, round_up, dy.device)
    return dy[:, oy][:, :, ox] / cnt[oy][:, ox][None, :, :, None].float()


# ------------------------------------------------------------------------------------------------
# SYMMETRIC pad
# ------------------------------------------------------------------------------------------------
def mirror_index(L, p, reflect=False):
    """source index of each of the L + 2p padded positions: tf.pad 'SYMMETRIC' repeats the edge (reflect=True: 'REFLECT', which
    does not, a negative control)"""
    i = torch.arange(-p, L + p)
    e = 0 if reflect else 1
    return torch.where(i < 0, -i - e, torch.where(i >= L, 2 * L - 1 - i - (1 - e), i))


def mirror_pad_ref(x, p, reflect=False):
    B, H, W, C = x.shape
    dev = x.device
    return x[:, mirror_index(H, p, reflect).to(dev)][:, :, mirror_index(W, p, reflect).to(dev)]


def _keep_but_third(L, p):
    """False at the padded position that is the third preimage of its source (one mirrored on both sides, 2p > L)"""
    j = torch.arange(L + 2 * p)
    s = mirror_index(L, p)
    return ~((s < p) & (s >= L - p) & (j >= p + L))


def mirror_pad_bwd_ref(dy, H, W, p, drop_third=False):
    """MirrorPadGrad: each dx element sums the padded positions that mirror onto it (up to 3 per axis) -> (dx fp64, magnitude
    sum|terms|, term count).  drop_third=True leaves out the third preimage of a row or column (a negative control)."""
    B, Hp, Wp, C = dy.shape
    dev = dy.device
    iy, ix = mirror_index(H, p).to(dev), mirror_index(W, p).to(dev)
    d = dy.double()
    one = torch.ones(1, Hp, Wp, 1, dtype=torch.float64, device=dev)
    if drop_third:
        keep = (_keep_but_third(H, p)[:, None] & _keep_but_third(W, p)[None, :]).to(dev)[None, :, :, None]
        d, one = d * keep, one * keep

    def fold(t):
        r = torch.zeros(t.shape[0], H, Wp, t.shape[3], dtype=torch.float64, device=dev).index_add_(1, iy, t)
        return torch.zeros(t.shape[0], H, W, t.shape[3], dtype=torch.float64, device=dev).index_add_(2, ix, r)

    return fold(d), fold(d.abs()), fold(one)


# ------------------------------------------------------------------------------------------------
# phase shift, discriminator input, logits | argmax
# ------------------------------------------------------------------------------------------------
def _ps_perm(order_b1, swap):
    # X viewed as [B, a, b, G, s1, s2] with sub = s1 * r + s2.  order_b1: sub = ry * r + rx; batch >= 2 order: sub = rx * r + ry
    b1 = bool(order_b1) != bool(swap)
    return (0, 1, 4, 2, 5, 3) if b1 else (0, 1, 5, 2, 4, 3)


def phase_shift_ref(X, r, G, order_b1, swap=False):
    """ops.PS of X [B, a, b, G*r*r] -> [B, a*r, b*r, G]: out[n, iy*r + ry, ix*r + rx, g] = X[n, iy, ix, g*r*r + sub] with
    sub = ry*r + rx in the batch_size == 1 order and rx*r + ry otherwise (swap=True exchanges them, a negative control)"""
    B, a, b, _ = X.shape
    return X.view(B, a, b, G, r, r).permute(*_ps_perm(order_b1, swap)).reshape(B, a * r, b * r, G)


def phase_shift_inv(Y, r, G, order_b1):
    """the inverse permutation: [B, a*r, b*r, G] -> [B, a, b, G*r*r]"""
    B, OH, OW, _ = Y.shape
    a, b = OH // r, OW // r
    # Y viewed as [B, a, ry, b, rx, G]
    perm = (0, 1, 3, 5, 2, 4) if order_b1 else (0, 1, 3, 5, 4, 2)
    return Y.reshape(B, a, r, b, r, G).permute(*perm).reshape(B, a, b, G * r * r)


def tile_channels(ps, ntile, blocked=False):
    """tf.tile along channels: [g0 .. g(G-1)] ntile times; blocked=True gives [g0 g0 g0 g1 ...] (a negative control)"""
    return ps.repeat_interleave(ntile, dim=3) if blocked else ps.repeat(1, 1, 1, ntile)


def phase_shift_fwd_ref(X, out0, r, G, coff, ntile, order_b1, swap=False, ignore_coff=False, blocked=False):
    """pnp_phase_shift_fwd into a copy of out0 [B, a*r, b*r, Ctot]: channels [coff, coff + ntile*G) are written, the rest kept"""
    out = out0.clone()
    c0 = 0 if ignore_coff else coff
    out[..., c0:c0 + ntile * G] = tile_channels(phase_shift_ref(X, r, G, order_b1, swap), ntile, blocked)
    return out


def phase_shift_bwd_ref(dout, r, G, coff, ntile, order_b1, drop_tiles=False):
    """pnp_phase_shift_bwd: dX = PS^-1 of the sum of the ntile copies (fp64); drop_tiles=True reads copy 0 only (a negative
    control)"""
    d = dout.double()
    s = sum(d[..., coff + t * G:coff + (t + 1) * G] for t in range(1 if drop_tiles else ntile))
    return phase_shift_inv(s, r, G, order_b1)


def argmax_first(l, last=False):
    """tf.argmax over the last axis: the lowest index among the maxima (last=True: the highest, a negative control)"""
    C = l.shape[-1]
    m = l.amax(-1, keepdim=True)
    k = torch.arange(C, device=l.device)
    if last:
        return torch.where(l == m, k, torch.full_like(k, -1)).amax(-1)
    return torch.where(l == m, k, torch.full_like(k, C)).amin(-1)


def disc_input_ref(srcs, Gs, ntiles, logits, r, order_b1, **bug):
    """adversarial.py:325-335 for any plan: [PS_r(src_0) tiled ntile_0 times | ... | logits | float(argmax logits)].
    bug: swap / blocked / last, the negative controls of the parts."""
    parts = [tile_channels(phase_shift_ref(s, r, G, order_b1, bug.get("swap", False)), t, bug.get("blocked", False))
             for s, G, t in zip(srcs, Gs, ntiles)]
    am = argmax_first(logits, bug.get("last", False)).to(logits.dtype).unsqueeze(-1)
    return torch.cat(parts + [logits, am], dim=3)


def logits_argmax_concat_ref(logits, out0, coff, last=False):
    """pnp_logits_argmax_concat into a copy of out0 [P, Ctot]: channels [coff, coff + C) = logits, coff + C = float(argmax)"""
    P, C = logits.shape
    out = out0.clone()
    out[:, coff:coff + C] = logits
    out[:, coff + C] = argmax_first(logits, last).to(out.dtype)
    return out


# ------------------------------------------------------------------------------------------------
# slice, concat, one-hot, fill
# ------------------------------------------------------------------------------------------------
def channel_slice_ref(g, C, off, Cs, out0, accumulate, ignore_acc=False):
    """out[m, 0:Cs] (+)= g[m, off:off+Cs]; the accumulation is one fp32 addition"""
    v = g.reshape(-1, C)[:, off:off + Cs]
    return out0 + v if (accumulate and not ignore_acc) else v.clone()


def crop_offsets(H1, W1, H2, W2, round_up=False):
    return ((H1 - H2 + 1) // 2, (W1 - W2 + 1) // 2) if round_up else ((H1 - H2) // 2, (W1 - W2) // 2)


def crop_concat_fwd_ref(x1, x2, round_up=False):
    """layers.py:108-115: [centre crop of x1 to x2's height and width | x2] along channels"""
    H2, W2 = x2.shape[1], x2.shape[2]
    oy, ox = crop_offsets(x1.shape[1], x1.shape[2], H2, W2, round_up)
    return torch.cat([x1[:, oy:oy + H2, ox:ox + W2], x2], dim=3)


def crop_concat_bwd_ref(dout, H1, W1, C1, round_up=False):
    """-> (dx1 [B, H1, W1, C1], +0 outside the crop; dx2)"""
    B, H2, W2, _ = dout.shape
    oy, ox = crop_offsets(H1, W1, H2, W2, round_up)
    dx1 = torch.zeros(B, H1, W1, C1, dtype=dout.dtype, device=dout.device)
    dx1[:, oy:oy + H2, ox:ox + W2] = dout[..., :C1]
    return dx1, dout[..., C1:].clone()


def one_hot_ref(labels, C, clamp=False):
    """lib._label_decomp: out[p, c] = (label[p] == c); a label outside [0, C) gives a zero row (clamp=True clamps it into
    range, a negative control)"""
    l = labels.clamp(0, C - 1) if clamp else labels
    return (l[:, None] == torch.arange(C, device=labels.device)[None, :]).float()


def fill_ref(buf, v, n, drop_tail=False):
    """pnp_fill into a copy of buf: the first n elements become v (drop_tail=True skips the last n % 4, a negative control)"""
    out = buf.clone()
    out[:(n // 4) * 4 if drop_tail else n] = v
    return out


# ------------------------------------------------------------------------------------------------
# the two transcendental kernels: fp64 references and a priori bounds
# ------------------------------------------------------------------------------------------------
# CUDA's documented maximum errors (CUDA C++ Programming Guide, "Mathematical Functions", single precision, default flags):
# expf 2 ulp, logf 1 ulp; +, *, / and fmaf are correctly rounded.  One ulp of a normal fp32 value v is at most 2u|v|.
EXPF_ULP, LOGF_ULP = 2, 1


def ps2_bound(C):
    """relative bound of pixel_softmax2's p_c = expf(l_c) / sum_c expf(l_c) (no max subtraction), for pixels whose exponentials
    are normal numbers: 2 ulp = 4u for the numerator's expf, 4u + (C - 1)u for the denominator (its expf's and C - 1
    additions of positive terms), u for the division: (C + 8)u to first order; gamma_{C+9} covers the higher-order terms"""
    return gamma(C + 9)


# cross_entropy_bwd: dy = k * logf(clip p) with k = -g / (float)n: 1 ulp = 2u for logf, u for k, u for the product
CE_DY_BOUND = gamma(2 * LOGF_ULP + 2)
# dp = (k * y) / p: u for k, u for the product, u for the division
CE_DP_BOUND = gamma(3)


def ce_acc_bound(n):
    """relative (to sum |y log clip p|) bound of cross_entropy_acc's sum: each thread accumulates at most CE_FLUSH terms with fmaf
    into an fp32 partial (gamma_32) of terms carrying logf's 2u, then fp64 additions (n * 2^-53 covers them generously)"""
    return gamma(CE_FLUSH + 2 * LOGF_ULP) + n * 2.0 ** -53


def ps2_special(logits):
    """pixels whose fp32 exponentials overflow (a logit above 88.73) or all underflow (every logit below -103.98): the kernel's
    quotient is inf/inf or 0/0 = NaN, which the +-1e15 clip turns into -1e15 (fmaxf drops the NaN)"""
    return (logits.amax(-1) > 88.73) | (logits.amax(-1) < -103.98)


def pixel_softmax2_ref(logits):
    """layers.py:134-138 in fp64: exp(l) / sum exp(l) over the last axis, no max subtraction"""
    e = torch.exp(logits.double())
    return e / e.sum(-1, keepdim=True)


def ce_clip(p):
    return p.double().clamp(CE_CLIP_LO, 1.0)


def cross_entropy_fwd_ref(y, p):
    """-> (sum y * log(clip(p, 1e-10f, 1)) in fp64, sum |y log clip p|)"""
    t = y.double() * torch.log(ce_clip(p))
    return t.sum(), t.abs().sum()


def cross_entropy_bwd_ref(y, p, g, n):
    """-> (dy, dp) in fp64 with k = -g / n exact: dy = k log(clip p); dp = k y / p where 1e-10f <= p <= 1, else 0"""
    k = -float(g) / n
    pd = p.double()
    dy = k * torch.log(ce_clip(p))
    inside = (pd >= CE_CLIP_LO) & (pd <= 1.0)
    dp = torch.where(inside, k * y.double() / torch.where(inside, pd, torch.ones_like(pd)), torch.zeros_like(pd))
    return dy, dp


def worst_ratio(got, ref, mag):
    r = (got.double() - ref.double()).abs() / mag.double().clamp_min(1e-300)
    r = torch.where(got.double() == ref.double(), torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0
