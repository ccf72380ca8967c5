"""The middle of ConvFeedForward / FeedForward (transformer.py:122-161) in float64, in the layouts of the FFN kernels;
shared by tests/test_ffn_reference_cpu.py and tests/test_ffn_reference_gpu.py.

For B sequences of N rows (M = B N) and F inner channels the kernels compute
  u    = xn W1^T                          [M, 2F]: value half u[:, :F], gate half u[:, F:]        (gemm_ffn_up)
  y[t] = w0 u[t-2] + w1 u[t-1] + w2 u[t]  per channel, zero history at every sequence start;
                                          y = u in the plain FeedForward (conv_w None)              (gemm_ffn_up)
  h    = gelu(y_gate) y_value             exact-erf GELU; row sums s1 = sum_c h, s2 = sum_c h^2    (gemm_ffn_up)
  hn   = (h - mean) rstd gamma keep / (1 - p)   bias-less LayerNorm over F, eps 1e-5; dropout     (ffn_norm_fwd)
and the backward pass maps d hn to du, dgamma and dconv_w                                           (ffn_mid_bwd)

Kernel layouts: u / du are [M, 2Fp] in the interleaved GEGLU order, 128-channel groups stored as [128 value | 128 gate]
columns; h / hn are [M, Fp]; Fp = F rounded up to a multiple of 128, padded columns zero.  The dropout keep mask is
[M, Fp/8] uint8, bit i of byte j = channel 8 j + i.  Everything here takes and returns the canonical [value F | gate F]
order; ileave_cols / to_kernel / from_kernel convert.

  forward(...)   every stage in float64.  u, h, stats: start that stage from the kernel's own stored upstream tensor
                 instead of the reference's, so that a test can tell one kernel's error from the rounding it inherits.
  grads(...)     du, dgamma, dconv_w by float64 autograd through forward().
  magnitude(...) componentwise scales S: the same passes on |.|, with bounds on GELU and its slope in place of GELU.
                 A kernel that rounds its stored result to a unit u errs by at most a few u times S, entry by entry.

Every function accepts any float dtype and device; the arithmetic is float64 on the inputs' device."""
import torch
import torch.nn.functional as nnf

EPS = 1e-5
GELU_SLOPE = 1.13       # max |gelu'(z)| = 1.1289 (at z = sqrt 2); also |gelu(z)| <= |z|


# ------------------------------------------------------------------------------------------------ layouts
def ileave_cols(F, device="cpu"):
    """Canonical column (value c | gate F + c) -> column of the interleaved [., 2Fp] layout."""
    c = torch.arange(F, device=device)
    a = (c // 128) * 256 + (c % 128)
    return torch.cat([a, a + 128])


def padded(F):
    return (F + 127) // 128 * 128


def to_kernel(x, F):
    """[..., 2F] canonical -> [..., 2Fp] interleaved, zeros in the padded columns."""
    out = x.new_zeros(*x.shape[:-1], 2 * padded(F))
    out[..., ileave_cols(F, x.device)] = x
    return out


def from_kernel(x, F):
    """[..., 2Fp] interleaved -> [..., 2F] canonical."""
    return x[..., ileave_cols(F, x.device)]


def unpack_keep(bits, F):
    """[M, Fp/8] uint8 keep bits (bit i of byte j = channel 8 j + i) -> [M, F] bool."""
    shifts = torch.arange(8, device=bits.device, dtype=torch.uint8)
    return ((bits[:, :, None] >> shifts) & 1).bool().reshape(bits.shape[0], -1)[:, :F]


def pack_keep(keep, Fp):
    """[M, F] bool -> [M, Fp/8] uint8 in ffn_norm_fwd's bit order (padded channels 0)."""
    M, F = keep.shape
    k = torch.zeros(M, Fp, dtype=torch.int32, device=keep.device)
    k[:, :F] = keep.int()
    return (k.view(M, Fp // 8, 8) << torch.arange(8, device=keep.device)).sum(-1).to(torch.uint8)


# ------------------------------------------------------------------------------------------------ forward
def conv(u, w, N):
    """Causal depthwise conv k = 3 over each sequence of N rows (transformer.py:122-131): y[t] = w0 u[t-2] + w1 u[t-1]
    + w2 u[t], rows before the sequence start are zero.  u [M, C], w [C, 3] or None (y = u)."""
    if w is None:
        return u
    M, C = u.shape
    up = nnf.pad(u.reshape(M // N, N, C), (0, 0, 2, 0))
    return (up[:, :-2] * w[:, 0] + up[:, 1:-1] * w[:, 1] + up[:, 2:] * w[:, 2]).reshape(M, C)


def conv_t(dy, w, N):
    """The transpose of conv: du[t] = w2 dy[t] + w1 dy[t+1] + w0 dy[t+2] within each sequence."""
    if w is None:
        return dy
    M, C = dy.shape
    dp = nnf.pad(dy.reshape(M // N, N, C), (0, 0, 0, 2))
    return (dp[:, :-2] * w[:, 2] + dp[:, 1:-1] * w[:, 1] + dp[:, 2:] * w[:, 0]).reshape(M, C)


def geglu(y):
    F = y.shape[-1] // 2
    return nnf.gelu(y[:, F:]) * y[:, :F]                       # transformer.py:134-137, exact erf


def forward(xn, W1, conv_w, gamma, N, keep=None, p=0.0, u=None, h=None, stats=None):
    """-> dict of float64 tensors: u [M, 2F], y [M, 2F], h [M, F] (= geglu(y), from u), s1 / s2 [M] (row sums of that
    h), mean / rstd [M], hhat [M, F], hn [M, F].

    u: the stored u (canonical order) to start from instead of xn W1^T (xn, W1 may then be None).  h: the stored h for
    the LayerNorm.  stats: (mean, rstd) to normalise with instead of the statistics of h.  keep: [M, F] bool or None."""
    w = None if conv_w is None else conv_w.double()
    u = xn.double() @ W1.double().t() if u is None else u.double()
    y = conv(u, w, N)
    hm = geglu(y)
    hl = hm if h is None else h.double()
    if stats is None:
        mean = hl.mean(-1)
        rstd = (((hl - mean[:, None]) ** 2).mean(-1) + EPS).rsqrt()
    else:
        mean, rstd = stats[0].double(), stats[1].double()
    hhat = (hl - mean[:, None]) * rstd[:, None]
    hn = hhat * gamma.double()
    if keep is not None:
        hn = hn * keep.double() / (1.0 - p)
    return {"u": u, "y": y, "h": hm, "s1": hm.sum(-1), "s2": (hm * hm).sum(-1), "mean": mean, "rstd": rstd,
            "hhat": hhat, "hn": hn}


def grads(u, conv_w, gamma, dhn, N, keep=None, p=0.0):
    """d sum(hn * dhn) by float64 autograd through forward() from u -> {"du" [M, 2F], "dgamma" [F], "dconv_w" [2F, 3] or
    None}.  LayerNorm statistics are recomputed from u, as the backward kernel's are (from the stored u)."""
    leaf = lambda t: None if t is None else t.detach().double().clone().requires_grad_(True)
    ul, wl, gl = leaf(u), leaf(conv_w), leaf(gamma)
    with torch.enable_grad():
        hn = forward(None, None, wl, gl, N, keep, p, u=ul)["hn"]
        hn.backward(dhn.double())
    return {"du": ul.grad, "dgamma": gl.grad, "dconv_w": None if wl is None else wl.grad}


def lnbwd_row_sums(dhn, hn, gamma, keep=None, p=0.0):
    """The LayerNorm-backward row sums the kernels form per 128-channel tile, over the first F channels of [M, Fp]
    inputs: s1 = sum gamma g (g = dropout-backward(dhn)), s2 = sum dhn hn -> [M, Fp/128] each."""
    M, Fp = dhn.shape
    F = gamma.shape[0]
    g = dhn.double()[:, :F]
    if keep is not None:
        g = g * keep.double() / (1.0 - p)
    s1 = torch.zeros(M, Fp, dtype=torch.float64, device=dhn.device)
    s1[:, :F] = gamma.double() * g
    s2 = dhn.double() * hn.double()
    return s1.view(M, -1, 128).sum(-1), s2.view(M, -1, 128).sum(-1)


# ------------------------------------------------------------------------------------------------ error scales
def magnitude(xn, W1, conv_w, gamma, N, keep=None, p=0.0, u=None, dhn=None, floor=0.0):
    """Componentwise scales of forward() and grads(), all float64 [same shapes as the tensors they scale]:

      u      |xn| |W1|^T  (|u| when the stage starts from a stored u)
      y      conv of S_u with |w|
      h      (1 + GELU_SLOPE) S_yg S_ya: an error e S_y in y moves h by at most e S_h, and |h| <= S_h
      s1, s2 sum_c S_h, sum_c 2 S_h^2
      mean   mean_c S_h
      var    2 mean_c(|h - mean| S_h)  (first order: d var = 2 mean_c((h - mean) dh)); var32 = mean_c(h^2) + mean^2, the
             scale of the fp32 one-pass E[h^2] - mean^2
      rstd   rstd^3 var / 2,  rstd32 = rstd^3 var32 / 2 + rstd
      hn     |gamma| keep/(1-p) (rstd (S_h + mean_c S_h + |hhat| mean_c(|hhat| S_h)) + |hhat|): an error e S_h in h moves
             hn by at most e S_hn (LayerNorm's row means included), and |hn| <= S_hn
    floor is added to the scales of the stored stages u, h and hn, and so carried through the later ones: a 16-bit store
    errs by at most unit |x| + tiny = unit (|x| + tiny / unit), tiny half the subnormal spacing (2^-25 in fp16, where
    2^-25 / 2^-11 = 2^-14 is the floor; bf16 has fp32's range and needs none).
    and given dhn (the backward from the stored u, so S_u = |u|):
      dh     rstd (|gamma g| + mean_c |gamma g| + |hhat| mean_c |gamma g hhat|)
      dy     value half S_dh |y_gate|, gate half GELU_SLOPE S_dh |y_value|
      du     the transposed conv of S_dy with |w|
      dgamma sum_t |g hhat|
      dconv_w  sum_t S_dy[t] |u[t - 2 + k]| for tap k"""
    aw = None if conv_w is None else conv_w.double().abs()
    su = (u.double().abs() if u is not None else xn.double().abs() @ W1.double().abs().t()) + floor
    sy = conv(su, aw, N)
    F = sy.shape[-1] // 2
    sh = (1.0 + GELU_SLOPE) * sy[:, F:] * sy[:, :F] + floor
    r = forward(xn, W1, conv_w, gamma, N, keep, p, u=u)
    h, mean, rstd, hhat = r["h"], r["mean"], r["rstd"], r["hhat"]
    ks = torch.ones_like(h) if keep is None else keep.double() / (1.0 - p)
    ag = gamma.double().abs()
    svar = 2 * ((h - mean[:, None]).abs() * sh).mean(-1)
    svar32 = (h * h).mean(-1) + mean * mean
    out = {"u": su, "y": sy, "h": sh, "s1": sh.sum(-1), "s2": 2 * (sh * sh).sum(-1), "mean": sh.mean(-1),
           "var": svar, "rstd": rstd ** 3 * svar / 2, "rstd32": rstd ** 3 * svar32 / 2 + rstd,
           "hn": ag * ks * (rstd[:, None] * (sh + sh.mean(-1, keepdim=True)
                                             + hhat.abs() * (hhat.abs() * sh).mean(-1, keepdim=True)) + hhat.abs())
                 + floor}
    if dhn is None:
        return out
    g = dhn.double() * ks
    agg = ag * g.abs()
    sdh = rstd[:, None] * (agg + agg.mean(-1, keepdim=True) + hhat.abs() * (agg * hhat.abs()).mean(-1, keepdim=True))
    y = r["y"]
    sdy = torch.cat([sdh * y[:, F:].abs(), GELU_SLOPE * sdh * y[:, :F].abs()], 1)
    out.update(dh=sdh, dy=sdy, du=conv_t(sdy, aw, N), dgamma=(g.abs() * hhat.abs()).sum(0))
    if aw is not None:
        M, C = su.shape
        up = nnf.pad(su.reshape(M // N, N, C), (0, 0, 2, 0))
        d = sdy.reshape(M // N, N, C)
        out["dconv_w"] = torch.stack([(d * up[:, k:k + N]).sum((0, 1)) for k in range(3)], 1)
    else:
        out["dconv_w"] = None
    return out
