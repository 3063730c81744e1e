"""Kernel-level tests of the per-sample attention kernels of the denoiser (denoiser.cu: k_attn_ln, k_xattn_ln,
k_attn_xattn_ln, the three k_qan_xattn_ln instantiations) and of the folded operands they consume, element by element
against float64 references of the kernels' contracts (include/interdiff_b200.h, idb_attn_desc).

Error model, per output element, u = 2^-24.  Operand terms rho / sigma as in test_gpu_gemm_kernels.py.

* Products.  Every product runs as mma.sync m16n8k16 on fp16 (hi, lo) pairs split on the fly (mma_pairs: hi*hi in the
  main accumulator, lo*hi + hi*lo in the small one, folded in with 2^-11).  mma.sync is assumed to round like a wgmma
  k-step: at most 2 ulp per instruction, i.e. 4u times the running sum of |a||w| through that k-step.  A product at k-step s
  of an accumulator that runs ns k-steps enters ns - s of them (weight 4 (ns - s)), the small accumulator (ns - s) / 127, the
  epilogue fmaf 1.  The self-attention logits are one accumulator over K = 64 (ns = 4), then * 1/8 (exact).  Cross-attention
  and QaN logits are 4 k-slices of 64 summed in the fixed order ((p0 + p1) + p2) + p3 (slice b enters 4 - max(b, 1) fp32
  additions), plus kc (u |logit|).  The value products run one accumulator over the HT16 <= 144 probabilities of all heads
  (ns = HT16 / 16, k index h * Tk + j).
* Softmax.  The kernels subtract the row maximum (u |l - max|, relative in exp), call expf (2 ulp), sum in fp32 (a warp tree
  of <= 6 levels), take one reciprocal (or division) and one product: relative c u with c = 10 (self / cross), 6 (QaN).  A
  logit error dl enters to first order as |dp_j| <= p_j (|dl_j| + max_k |dl_k|).  The probabilities are then re-split into
  pairs: their representation error is the rho term of the value product, and the kernel's dp goes through |V|.
* QaN taps.  c_s = sum_n wk_n a_ns is a 32-lane warp sum (5u of sum |wk_n a_ns|); the 3-tap filter is one product and two
  fmaf (3u of sum_s |c_s x_s|); the residual x + y one rounding.
* Bias and residual.  u |result| per fp32 addition.
* LayerNorm.  First order in the input error dz:  |dy_n| <= |w_n| rstd (|dz_n| + mean|dz| + |x^_n| mean(|x^||dz|)).  Its own
  rounding enters the same way: the mean of 256 values (8 per lane, then 5 shuffle levels) is off by <= 12u mean|z|, the
  centring by u |z_n - mean|, rstd by 12u relative (variance sum, sqrt, reciprocal, the product with rstd), the closing
  fmaf by u |y|.  The pending norm of a QaN layer is a LayerNorm of exact input rows: its own rounding is the input error of
  the QaN block.

All terms above are first order; second-order terms (products of two u-sized errors, exp(dl) - 1 - dl for |dl| < 1e-4) are
below 1 % of the bound and covered by a factor 1.01 (SLACK).  The bound is worst case; each case records its largest
err / bound as the `ratio` property.  It discriminates: with the operands and probabilities of the kernel's arithmetic
carried as single fp16 values (lo terms dropped) or with the QaN slot mask off by one at t = T-1, the float64 emulation
exceeds the bound by far more than 4x (test_bound_detects_*; they run on the CPU).

The decoder QaN kernels keep their LN1 rows in shared memory, so the composed bound carries the LN1 bound through the
cross-attention logits as sum |dx1||kp|, which is loose.  Their output is also checked against the cross-attention bound
on the rows the encoder variant computes from the same operands (same code, `_given_x1`), which is as tight as the other
kernels' bounds.

Kernel names appear in every case ID: test_attn_ln, test_xattn_ln, test_attn_xattn_ln, and in test_qan's parameters
qan_xattn_ln_pre = k_qan_xattn_ln<true, true>, qan_xattn_ln = <true, false>, qan_ln / qan_ln_pre = <false> (pending norm off /
on).
"""
import math

import pytest
import torch

from tests.test_gpu_gemm_kernels import U, rho, sigma, simt_bound, tc_bound

D, H, HD = 256, 4, 64
SLACK = 1.01
SENT = -7.777e33
gpu = pytest.mark.gpu
HAS_GPU = torch.cuda.is_available()
DEV = "cuda:0" if HAS_GPU else "cpu"


# ------------------------------------------------------------------ float64 references and bounds
def mma_weights(K, slices, dev):
    """per-k weight (in u) of a product through the pair products of a kernel: `slices` accumulators of K / slices
    summed in a fixed order"""
    k = torch.arange(K, device=dev)
    per = K // slices
    sl, s = k // per, (k % per) // 16
    ns = -(-per // 16)
    w = 4.0 * (ns - s) + (ns - s) / 127.0 + 1.0
    if slices > 1:
        w = w + (slices - torch.clamp(sl, min=1))
    return w.double()


def mma_bound(A, B, slices=1):
    """element-wise bound on |A @ B - C| of the kernel's product, A [.., M, K], B [.., K, N] exact float64 operands that the
    kernel splits into pairs on the fly"""
    w = mma_weights(A.shape[-1], slices, A.device)
    aA, aB = A.abs(), B.abs()
    return (U * ((aA * w) @ aB) + sigma(A) @ sigma(B) + rho(A) @ aB + aA @ rho(B) + 2.0 ** -46 * (aA @ aB))


def softmax_bound(l, el, valid, c):
    """float64 softmax over the last dim where `valid`, and the bound of the module docstring given the logit bound el"""
    lm = l.masked_fill(~valid, -math.inf)
    m = lm.max(dim=-1, keepdim=True).values
    p = torch.softmax(lm, dim=-1)
    el = el.masked_fill(~valid, 0)
    ep = p * (el + el.max(dim=-1, keepdim=True).values) + p * U * (c + (l - m).abs().masked_fill(~valid, 0))
    return p, ep


def layer_norm(z, ez, w, b):
    """float64 LayerNorm (eps 1e-5) of rows z and the bound of the module docstring given the input bound ez"""
    w, b = w.double(), b.double()
    mu = z.mean(dim=-1, keepdim=True)
    c = z - mu
    rstd = 1.0 / torch.sqrt((c * c).mean(dim=-1, keepdim=True) + 1e-5)
    xh = c * rstd
    y = xh * w + b
    dc = ez + ez.mean(dim=-1, keepdim=True) + 12 * U * z.abs().mean(dim=-1, keepdim=True) + U * c.abs()
    rr = rstd * (xh.abs() * dc).mean(dim=-1, keepdim=True) + 12 * U
    return y, SLACK * (w.abs() * rstd * dc + (w * xh).abs() * rr) + U * y.abs()


def add_round(y, e, x):
    y = y + x.double()
    return y, e + U * y.abs()


def ref_self(q, k, v, res, bo, ln, B, T):
    """self-attention + LN1: q, k [B*T, >= 256], v [B*T, >= H*256]; returns the output [B*T, 256] and its bound"""
    q = q[:B * T, :D].double().reshape(B, T, H, HD).permute(0, 2, 1, 3)
    k = k[:B * T, :D].double().reshape(B, T, H, HD).permute(0, 2, 1, 3)
    v = v[:B * T, :H * D].double().reshape(B, T, H, D).permute(0, 2, 1, 3).reshape(B, H * T, D)
    l = q @ k.transpose(-1, -2) / 8
    el = mma_bound(q, k.transpose(-1, -2)) / 8
    p, ep = softmax_bound(l, el, torch.ones_like(l, dtype=torch.bool), 10)
    P = p.permute(0, 2, 1, 3).reshape(B, T, H * T)
    EP = ep.permute(0, 2, 1, 3).reshape(B, T, H * T)
    y = P @ v
    e = EP @ v.abs() + mma_bound(P, v)
    y, e = add_round(y, e, bo)
    y, e = add_round(y, e, res[:B * T].reshape(B, T, D))
    y, e = layer_norm(y, e, *ln)
    return y.reshape(B * T, D), e.reshape(B * T, D)


def ref_cross(x1, ex1, kp, vp, kc, bo2, ln2, B, T, Tk):
    """cross-attention + LN2 on rows x1 [B*T, 256] (bound ex1 or None); memory rows j*B + b"""
    x = x1[:B * T].double().reshape(B, T, D)
    ex = ex1.reshape(B, T, D) if ex1 is not None else torch.zeros_like(x)
    kpb = kp.double().reshape(Tk, B, H, D).permute(1, 2, 0, 3).reshape(B, H * Tk, D)
    vpb = vp.double().reshape(Tk, B, H, D).permute(1, 2, 0, 3).reshape(B, H * Tk, D)
    kcb = kc.double().reshape(Tk, B, H).permute(1, 2, 0).reshape(B, 1, H * Tk)
    l = x @ kpb.transpose(-1, -2) + kcb
    el = mma_bound(x, kpb.transpose(-1, -2), slices=4) + U * l.abs() + ex @ kpb.abs().transpose(-1, -2)
    l4, el4 = l.reshape(B, T, H, Tk), el.reshape(B, T, H, Tk)
    p, ep = softmax_bound(l4, el4, torch.ones_like(l4, dtype=torch.bool), 10)
    P, EP = p.reshape(B, T, H * Tk), ep.reshape(B, T, H * Tk)
    y = P @ vpb
    e = EP @ vpb.abs() + mma_bound(P, vpb)
    y, e = add_round(y, e, bo2)
    y, e = add_round(y, e + ex, x)
    y, e = layer_norm(y, e, *ln2)
    return y.reshape(B * T, D), e.reshape(B * T, D)


def ref_qan(zin, pre, qt, wk, ln1, B, T, N, mask_shift=0):
    """QaN block + residual + LN1 on rows zin [B*T, 256] (optional pending norm `pre`); mask_shift = 1 emulates the slot
    mask off by one at the end of the window (slot 2 dropped at t = T-2 instead of t = T-1)"""
    x = zin[:B * T].double().reshape(B, T, D)
    ex = torch.zeros_like(x)
    if pre is not None:
        x, ex = layer_norm(x, ex, *pre)
    qt = qt.double().reshape(3, N, D)
    wk = wk.double().reshape(N)
    pad = torch.zeros(B, 1, D, dtype=x.dtype, device=x.device)
    xs = torch.cat([pad, x, pad], dim=1)
    es = torch.cat([pad, ex, pad], dim=1)
    src = [xs[:, s:s + T] for s in range(3)]                 # slot s of row t reads row t + s - 1
    esrc = [es[:, s:s + T] for s in range(3)]
    l = torch.stack([src[s] @ qt[s].T for s in range(3)], dim=-1)                         # [B, T, N, 3]
    el = torch.stack([mma_bound(src[s], qt[s].T, slices=4) + esrc[s] @ qt[s].abs().T for s in range(3)], dim=-1)
    t = torch.arange(T, device=x.device)
    valid = torch.stack([t > 0, torch.ones_like(t, dtype=torch.bool), t < T - 1 - mask_shift], dim=-1)
    valid = valid[None, :, None, :].expand(B, T, N, 3)
    a, ea = softmax_bound(l, el, valid, 6)
    c = torch.einsum("n,btns->bts", wk, a)
    ec = torch.einsum("n,btns->bts", wk.abs(), ea) + 5 * U * torch.einsum("n,btns->bts", wk.abs(), a)
    y = sum(c[..., s:s + 1] * src[s] for s in range(3))
    ey = sum(ec[..., s:s + 1] * src[s].abs() + c[..., s:s + 1].abs() * esrc[s] for s in range(3))
    ey = ey + 3 * U * sum((c[..., s:s + 1] * src[s]).abs() for s in range(3))
    v, ev = add_round(y, ey + ex, x)
    o, eo = layer_norm(v, ev, *ln1)
    return o.reshape(B * T, D), eo.reshape(B * T, D)


def check(record_property, got, want, bound, tag=""):
    err = (got.double() - want).abs()
    ratio = torch.where(err == 0, 0.0, err / bound).max().item()       # exact zeros (padding of the folded bias) have bound 0
    record_property("ratio" + tag, ratio)
    assert torch.isfinite(got).all(), tag
    assert ratio <= 1.0, (tag, ratio)
    return ratio


# ------------------------------------------------------------------ operands
def gen(seed, dev=DEV):
    return torch.Generator(device=dev).manual_seed(seed)


def ln_params(g, dev=DEV):
    return 1 + 0.1 * torch.randn(D, generator=g, device=dev), 0.1 * torch.randn(D, generator=g, device=dev)


def ln_rows(x):
    """LayerNorm'd rows (norm about 16), as the kernels see them in the model"""
    return torch.nn.functional.layer_norm(x, (D,))


def self_operands(family, B, T, seed, dev=DEV):
    """q, k, v' as views of one [B*T, 1536] projection buffer (the decoder's layout), residual, bo, ln1"""
    g = gen(seed, dev)
    M = B * T
    qkv = torch.randn(M, 2 * D + H * D, generator=g, device=dev)
    qkv[:, 2 * D:] /= math.sqrt(T)
    res = torch.randn(M, D, generator=g, device=dev)
    bo = 0.1 * torch.randn(D, generator=g, device=dev)
    ln = ln_params(g, dev)
    if family == "peaked":                  # logits up to about +-80, exact ties
        qkv[:, :2 * D] *= 5
        kk = qkv[:, D:2 * D].view(B, T, D)
        if T > 2:
            kk[:, T - 1] = kk[:, 0]                          # two keys with identical logits for every query
        qkv[1:M:3, :D] = 0                                   # queries with all logits 0 (a tie over every key)
    elif family == "offset":                # LayerNorm input 300 + O(0.05)
        qkv[:, 2 * D:] *= 0.01
        res = 300 + 0.05 * torch.randn(M, D, generator=g, device=dev)
    elif family == "tiny":                  # products near the fp16 subnormal floor
        qkv *= 2.0 ** -12
        res *= 2.0 ** -16
    return qkv, res, bo, ln


def views(qkv):
    return qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]


def memory_operands(family, B, Tk, seed, dev=DEV):
    g = gen(seed, dev)
    kp = torch.randn(Tk * B, H * D, generator=g, device=dev) / 16
    vp = torch.randn(Tk * B, H * D, generator=g, device=dev) / math.sqrt(H * Tk)
    kc = 0.5 * torch.randn(Tk * B, H, generator=g, device=dev)
    if family == "peaked":
        kp *= 5
        kc *= 10
        if Tk > 1:
            kp.view(Tk, B, H * D)[Tk - 1] = kp.view(Tk, B, H * D)[0]
            kc.view(Tk, B, H)[Tk - 1] = kc.view(Tk, B, H)[0]
    bo2 = 0.1 * torch.randn(D, generator=g, device=dev)
    return kp, vp, kc, bo2, ln_params(g, dev)


def qan_operands(family, B, T, N, seed, dev=DEV):
    g = gen(seed, dev)
    zin = ln_rows(torch.randn(B * T, D, generator=g, device=dev))
    qt = torch.randn(3 * N, D, generator=g, device=dev) / (16 * 16)     # norm 1/16 folded queries: logits ~ +-0.25
    if family == "peaked":
        qt *= 80
        qt[N - 1] = qt[0]                                                # tied slot-0 logits of queries 0 and N-1
        zin.view(B, T, D)[:, 1::2] = zin.view(B, T, D)[:, 0:1]           # repeated rows: tied slots
    elif family == "offset":
        zin = 300 + 0.05 * torch.randn(B * T, D, generator=g, device=dev)
        qt /= 300
    wk = torch.randn(N, 1, generator=g, device=dev)
    return zin, qt, wk, ln_params(g, dev), ln_params(g, dev)


# ------------------------------------------------------------------ engine plumbing
@pytest.fixture(scope="module")
def eng():
    from interdiff_b200.engine import Engine
    e = Engine(DEV)
    yield e
    e.close()


def outputs(B, T):
    out = torch.full((B * T + 40, D), SENT, device=DEV)
    hi = torch.full((B * T + 40, D), -1234.0, dtype=torch.float16, device=DEV)
    lo = torch.full_like(hi, 4320.0)
    return out, (hi, lo)


def split(eng, x):
    hi, lo = torch.empty(x.shape, dtype=torch.float16, device=DEV), torch.empty(x.shape, dtype=torch.float16, device=DEV)
    eng._chk(eng.lib.idb_debug_split(eng._h, eng._ptr(x), eng._ptr(hi), eng._ptr(lo), x.shape[0], x.shape[1], x.shape[1], eng._stream()))
    return hi, lo


def check_untouched_and_pairs(eng, out, pair, M):
    """rows >= M keep their canary values; the pair outputs are the library's split of the fp32 output, bit for bit"""
    assert bool((out[M:] == SENT).all()) and bool((pair[0][M:] == -1234.0).all()) and bool((pair[1][M:] == 4320.0).all())
    want = split(eng, out[:M].contiguous())
    assert torch.equal(pair[0][:M].view(torch.int16), want[0].view(torch.int16))
    assert torch.equal(pair[1][:M].view(torch.int16), want[1].view(torch.int16))


def run_self(eng, qkv, res, bo, ln, B, T, **kw):
    q, k, v = views(qkv)
    out, pair = outputs(B, T)
    eng.attention("attn_ln", B, T, q=q, k=k, v=v, res=res, bo=bo, ln1=ln, out=out, out_pair=pair, **kw)
    check_untouched_and_pairs(eng, out, pair, B * T)
    return out[:B * T]


def run_cross(eng, x1, mem, B, T, Tk, **kw):
    kp, vp, kc, bo2, ln2 = mem
    out, pair = outputs(B, T)
    eng.attention("xattn_ln", B, T, Tk, x1=x1, kp=kp, vp=vp, kc=kc, bo2=bo2, ln2=ln2, out=out, out_pair=pair, **kw)
    check_untouched_and_pairs(eng, out, pair, B * T)
    return out[:B * T]


def run_qan(eng, kernel, zin, pre, qt, wk, ln1, B, T, N, mem=None, Tk=0, **kw):
    out, pair = outputs(B, T)
    m = dict(kp=mem[0], vp=mem[1], kc=mem[2], bo2=mem[3], ln2=mem[4]) if mem is not None else {}
    eng.attention(kernel, B, T, Tk, N, zin=zin, pre=pre, qt=qt, wk=wk, ln1=ln1, out=out, out_pair=pair, **m, **kw)
    check_untouched_and_pairs(eng, out, pair, B * T)
    return out[:B * T]


# ------------------------------------------------------------------ 1. self-attention (k_attn_ln)
SELF_T = [1, 2, 8, 9, 16, 17, 32, 33, 36]
SELF_CASES = [(T, B, "normal") for T in SELF_T for B in (1, 3)] + [(30, 64, "normal")] + \
    [(T, 3, f) for f in ("peaked", "offset", "tiny") for T in (2, 17, 36)]


@gpu
@pytest.mark.parametrize("T,B,family", SELF_CASES)
def test_attn_ln(eng, record_property, T, B, family):
    qkv, res, bo, ln = self_operands(family, B, T, 100 * T + B)
    got = run_self(eng, qkv, res, bo, ln, B, T)
    want, bnd = ref_self(*views(qkv), res, bo, ln, B, T)
    check(record_property, got, want, bnd)


# ------------------------------------------------------------------ 2. cross-attention (k_xattn_ln)
CROSS_TK = [1, 2, 3, 8, 9, 15, 16]
CROSS_CASES = [(Tk, "normal") for Tk in CROSS_TK] + [(Tk, "peaked") for Tk in (1, 9, 16)]


@gpu
@pytest.mark.parametrize("Tk,family", CROSS_CASES)
def test_xattn_ln(eng, record_property, Tk, family):
    B, T = 3, 17
    x1 = ln_rows(torch.randn(B * T, D, generator=gen(Tk), device=DEV))
    mem = memory_operands(family, B, Tk, 7 * Tk)
    got = run_cross(eng, x1, mem, B, T, Tk)
    want, bnd = ref_cross(x1, None, *mem, B, T, Tk)
    check(record_property, got, want, bnd)


# ------------------------------------------------------------------ 3. fused standard layer (k_attn_xattn_ln)
FUSED_CASES = [(1, 1, 1), (3, 17, 9), (3, 36, 16), (64, 30, 10), (2, 9, 3)]


@gpu
@pytest.mark.parametrize("B,T,Tk", FUSED_CASES)
def test_attn_xattn_ln(eng, record_property, B, T, Tk):
    """bound on both halves, and bit-identity with k_attn_ln followed by k_xattn_ln (LN1 rows included)"""
    qkv, res, bo, ln = self_operands("normal", B, T, 3 * T + Tk)
    mem = memory_operands("normal", B, Tk, T)
    kp, vp, kc, bo2, ln2 = mem
    q, k, v = views(qkv)
    out, pair = outputs(B, T)
    x1 = torch.full((B * T + 40, D), SENT, device=DEV)
    eng.attention("attn_xattn_ln", B, T, Tk, q=q, k=k, v=v, res=res, bo=bo, ln1=ln, kp=kp, vp=vp, kc=kc, bo2=bo2, ln2=ln2,
                  out=out, out_pair=pair, x1_out=x1)
    check_untouched_and_pairs(eng, out, pair, B * T)
    assert bool((x1[B * T:] == SENT).all())
    x1 = x1[:B * T]
    want1, b1 = ref_self(q, k, v, res, bo, ln, B, T)
    check(record_property, x1, want1, b1, "_x1")
    want2, b2 = ref_cross(x1, None, *mem, B, T, Tk)
    check(record_property, out[:B * T], want2, b2)
    sep1 = run_self(eng, qkv, res, bo, ln, B, T)
    sep2 = run_cross(eng, sep1, mem, B, T, Tk)
    assert torch.equal(sep1, x1) and torch.equal(sep2, out[:B * T])


# ------------------------------------------------------------------ 4. QaN layers
QAN_T = [1, 2, 3, 16, 17, 18, 33, 36]
QAN_KERNELS = ["qan_xattn_ln_pre", "qan_xattn_ln", "qan_ln", "qan_ln_pre"]
QAN_CASES = [(kern, T, N, "normal") for kern in QAN_KERNELS for T in QAN_T for N in (10, 3)] + \
    [(kern, T, 10, f) for kern in ("qan_xattn_ln", "qan_ln_pre") for f in ("peaked", "offset") for T in (2, 17, 36)]


def qan_case(kern, B, T, N, family, seed):
    zin, qt, wk, ln1, pre = qan_operands(family, B, T, N, seed)
    with_pre = kern.endswith("_pre")
    kernel = "qan_ln" if kern.startswith("qan_ln") else kern
    if with_pre and family != "offset":
        zin = 3 + 2 * zin                       # something for the pending norm to undo
    return kernel, zin, (pre if with_pre else None), qt, wk, ln1


def check_qan_decoder(eng, record_property, got, zin, pre, qt, wk, ln1, mem, B, T, N, Tk):
    """a decoder QaN kernel's output against the composed bound (QaN block, LN1, cross-attention, LN2), and - much tighter -
    against the cross-attention bound on the LN1 rows the encoder variant computes from the same operands (the decoder
    variants run the same code on them before their cross-attention block; the rows never leave shared memory)"""
    want, bnd = ref_qan(zin, pre, qt, wk, ln1, B, T, N)
    want, bnd = ref_cross(want, bnd, *mem, B, T, Tk)
    check(record_property, got, want, bnd)
    x1 = eng.attention("qan_ln", B, T, 0, N, zin=zin, pre=pre, qt=qt, wk=wk, ln1=ln1)
    want, bnd = ref_cross(x1, None, *mem, B, T, Tk)
    check(record_property, got, want, bnd, "_given_x1")


@gpu
@pytest.mark.parametrize("kern,T,N,family", QAN_CASES)
def test_qan(eng, record_property, kern, T, N, family):
    B, Tk = 3, 5
    kernel, zin, pre, qt, wk, ln1 = qan_case(kern, B, T, N, family, 11 * T + N)
    if kernel == "qan_ln":
        got = run_qan(eng, kernel, zin, pre, qt, wk, ln1, B, T, N)
        check(record_property, got, *ref_qan(zin, pre, qt, wk, ln1, B, T, N))
        return
    mem = memory_operands("normal", B, Tk, T)
    got = run_qan(eng, kernel, zin, pre, qt, wk, ln1, B, T, N, mem, Tk)
    check_qan_decoder(eng, record_property, got, zin, pre, qt, wk, ln1, mem, B, T, N, Tk)


# ------------------------------------------------------------------ 5. the library's own operands (family `model`)
@pytest.fixture(scope="module")
def model(eng):
    from tests.helpers import mdm_weights
    sd = mdm_weights("smpl", "auto")
    eng.load_denoiser(sd, "smpl")
    B, T, Tk = 3, 30, 10
    cond = torch.randn(Tk, B, D, generator=torch.Generator().manual_seed(5))
    eng.bind(cond, T)
    return sd, B, T, Tk


def model_memory(eng, sd, layer):
    p = "decoder.layers.%d." % layer
    return (eng.denoiser_tensor(layer, "kp"), eng.denoiser_tensor(layer, "vp"), eng.denoiser_tensor(layer, "kc"),
            sd[p + "multihead_attn.out_proj.bias"].to(DEV), (sd[p + "norm2.weight"].to(DEV), sd[p + "norm2.bias"].to(DEV)))


@gpu
@pytest.mark.parametrize("kernel", ["attn_ln", "attn_xattn_ln"])
def test_model_standard_layer(eng, model, record_property, kernel):
    sd, B, T, Tk = model
    p = "decoder.layers.0."
    x = ln_rows(torch.randn(B * T, D, generator=gen(1), device=DEV))
    qkv = x @ eng.denoiser_tensor(0, "qkvf_w").T + eng.denoiser_tensor(0, "qkvf_b")
    bo, ln = eng.denoiser_tensor(0, "bo_f"), (sd[p + "norm1.weight"].to(DEV), sd[p + "norm1.bias"].to(DEV))
    want, bnd = ref_self(*views(qkv), x, bo, ln, B, T)
    if kernel == "attn_ln":
        check(record_property, run_self(eng, qkv, x, bo, ln, B, T), want, bnd)
        return
    mem = model_memory(eng, sd, 0)
    x1 = torch.empty(B * T, D, device=DEV)
    q, k, v = views(qkv)
    out = eng.attention(kernel, B, T, Tk, q=q, k=k, v=v, res=x, bo=bo, ln1=ln, kp=mem[0], vp=mem[1], kc=mem[2], bo2=mem[3],
                        ln2=mem[4], x1_out=x1)
    check(record_property, x1, want, bnd, "_x1")
    want2, bnd2 = ref_cross(x1, None, *mem, B, T, Tk)
    check(record_property, out, want2, bnd2)


@gpu
@pytest.mark.parametrize("kern", ["qan_xattn_ln_pre", "qan_xattn_ln"])
def test_model_qan_layer(eng, model, record_property, kern):
    sd, B, T, Tk = model
    layer = 1
    p = "decoder.layers.%d." % layer
    N = 10
    zin = ln_rows(torch.randn(B * T, D, generator=gen(2), device=DEV))
    pre = (sd["decoder.layers.0.norm3.weight"].to(DEV), sd["decoder.layers.0.norm3.bias"].to(DEV)) if kern.endswith("_pre") else None
    if pre is not None:
        zin = 3 + 2 * zin
    qt, wk = eng.denoiser_tensor(layer, "qt"), sd[p + "wk"].to(DEV)
    ln1 = (sd[p + "norm1.weight"].to(DEV), sd[p + "norm1.bias"].to(DEV))
    mem = model_memory(eng, sd, layer)
    got = run_qan(eng, kern, zin, pre, qt, wk, ln1, B, T, N, mem, Tk)
    check_qan_decoder(eng, record_property, got, zin, pre, qt, wk, ln1, mem, B, T, N, Tk)


# ------------------------------------------------------------------ 6. properties beyond the bound
@gpu
@pytest.mark.parametrize("kernel", ["attn_ln", "xattn_ln", "attn_xattn_ln", "qan_xattn_ln_pre", "qan_xattn_ln", "qan_ln"])
def test_sample_isolation_and_pdl(eng, kernel):
    """NaN in every row and memory slot of the other samples leaves sample b finite and bit-identical; programmatic
    dependent launch on and off give the same bits"""
    B, T, Tk, N, b = 3, 17, 9, 10, 1
    qkv, res, bo, ln = self_operands("normal", B, T, 1)
    kp, vp, kc, bo2, ln2 = memory_operands("normal", B, Tk, 2)
    zin, qt, wk, ln1q, pre = qan_operands("normal", B, T, N, 3)
    x1 = ln_rows(torch.randn(B * T, D, generator=gen(4), device=DEV))

    def launch(poison, pdl):
        ops = [t.clone() for t in (qkv, res, x1, zin, kp, vp, kc)]
        if poison:
            for t in ops[:4]:
                t.view(B, T, -1)[torch.arange(B, device=DEV) != b] = float("nan")
            for t in ops[4:]:
                t.view(Tk, B, -1)[:, torch.arange(B, device=DEV) != b] = float("nan")
        q, k, v = views(ops[0])
        kw = dict(q=q, k=k, v=v, res=ops[1], bo=bo, ln1=ln, x1=ops[2], kp=ops[4], vp=ops[5], kc=ops[6], bo2=bo2, ln2=ln2)
        if kernel.startswith("qan"):
            kw = dict(zin=ops[3], qt=qt, wk=wk, ln1=ln1q, pre=pre if kernel != "qan_xattn_ln" else None,
                      **({} if kernel == "qan_ln" else dict(kp=ops[4], vp=ops[5], kc=ops[6], bo2=bo2, ln2=ln2)))
        if kernel == "attn_xattn_ln":
            kw["x1_out"] = torch.empty(B * T, D, device=DEV)
        return eng.attention(kernel, B, T, 0 if kernel in ("attn_ln", "qan_ln") else Tk, N if kernel.startswith("qan") else 0,
                             pdl=pdl, **kw).view(B, T, D)

    clean = launch(False, False)
    assert torch.isfinite(clean).all()
    assert torch.equal(launch(False, True), clean)
    poisoned = launch(True, True)
    assert torch.isfinite(poisoned[b]).all() and torch.equal(poisoned[b], clean[b])


@gpu
def test_hook_rejects_unsupported_arguments(eng):
    from interdiff_b200.engine import EngineError
    qkv, res, bo, ln = self_operands("normal", 1, 37, 1)
    kp, vp, kc, bo2, ln2 = memory_operands("normal", 1, 17, 2)
    zin, qt, wk, ln1, pre = qan_operands("normal", 1, 8, 11, 3)
    q, k, v = views(qkv)
    x1 = zin
    bad = [
        lambda: eng.attention("attn_ln", 1, 37, q=q, k=k, v=v, res=res, bo=bo, ln1=ln),                        # T > 36
        lambda: eng.attention("xattn_ln", 1, 8, 17, x1=x1, kp=kp, vp=vp, kc=kc, bo2=bo2, ln2=ln2),              # Tk > 16
        lambda: eng.attention("xattn_ln", 1, 8, 0, x1=x1, kp=kp, vp=vp, kc=kc, bo2=bo2, ln2=ln2),               # Tk == 0
        lambda: eng.attention("qan_xattn_ln", 1, 8, 0, 10, zin=zin, qt=qt[:30], wk=wk[:10], ln1=ln1, kp=kp, vp=vp, kc=kc,
                              bo2=bo2, ln2=ln2),                                                                 # Tk == 0
        lambda: eng.attention("qan_ln", 1, 8, 0, 11, zin=zin, qt=qt, wk=wk, ln1=ln1),                           # N > 10
        lambda: eng.attention("attn_ln", 1, 8, q=q, k=k, v=v, res=res, bo=bo, ln1=ln, H=8),                     # H != 4
    ]
    n0 = eng.launch_count
    for i, f in enumerate(bad):
        with pytest.raises(EngineError, match="supported"):
            f()
    assert eng.launch_count == n0


# ------------------------------------------------------------------ 7. the bound discriminates (float64 emulations, CPU)
def f16(x):
    return x.half().double()


def test_bound_detects_single_fp16_arithmetic():
    """self-attention with q, k, v' and the probabilities carried as single fp16 values (the pairs' lo terms dropped),
    float64 otherwise: at least 4x over the bound"""
    B, T = 2, 17
    qkv, res, bo, ln = self_operands("normal", B, T, 5, dev="cpu")
    q, k, v = (f16(t).reshape(B, T, -1) for t in views(qkv))
    qh, kh = q.reshape(B, T, H, HD).transpose(1, 2), k.reshape(B, T, H, HD).transpose(1, 2)
    p = f16(torch.softmax(qh @ kh.transpose(-1, -2) / 8, dim=-1)).transpose(1, 2).reshape(B, T, H * T)
    vv = v.reshape(B, T, H, D).transpose(1, 2).reshape(B, H * T, D)
    z = p @ vv + bo.double() + res.double().reshape(B, T, D)
    y = torch.nn.functional.layer_norm(z, (D,), ln[0].double(), ln[1].double()).reshape(B * T, D)
    want, bnd = ref_self(*views(qkv), res, bo, ln, B, T)
    ratio = ((y - want).abs() / bnd).max().item()
    assert ratio > 4, ratio


def test_bound_detects_qan_mask_off_by_one():
    B, T, N = 2, 17, 10
    zin, qt, wk, ln1, _ = qan_operands("normal", B, T, N, 6, dev="cpu")
    want, bnd = ref_qan(zin, None, qt, wk, ln1, B, T, N)
    bad, _ = ref_qan(zin, None, qt, wk, ln1, B, T, N, mask_shift=1)
    ratio = ((bad - want).abs() / bnd).max().item()
    assert ratio > 4, ratio


# ------------------------------------------------------------------ 8. folded operands
def fold_reference(sd, layer, rotary, N=10):
    """float64 folds of the unfolded state_dict: (qkvf_w, qkvf_b, bo_f) of a standard layer or qt of a QaN layer"""
    p = "decoder.layers.%d." % layer
    f = lambda n: torch.as_tensor(sd[p + n]).double()
    if p + "queries" in sd:
        q = f("queries").reshape(N, H, HD)
        q = q / (q.norm(dim=-1, keepdim=True) + 1e-6) / math.sqrt(HD) * D ** -0.5
        q = q.reshape(N, D)
        # float32 frequencies, as the reference rotates with: the float32 roundings of the exact 10000^(-2i/256) (the
        # reference's torch-evaluated buffer differs from them by one ulp at 42 of the 128, DESIGN.md section 5)
        inv = (1.0 / 10000.0 ** (torch.arange(0, D, 2, dtype=torch.float64) / D)).float().double()
        from oracle.restate import ROTARY_OFFSETS
        out, terms = [], []
        for o in ROTARY_OFFSETS[rotary]:
            cs, sn = torch.cos(o * inv), torch.sin(o * inv)
            a, b = q[:, :D // 2], q[:, D // 2:]
            out.append(torch.cat([a * cs - b * sn, b * cs + a * sn], dim=1))
            terms.append(torch.cat([(a * cs).abs() + (b * sn).abs(), (b * cs).abs() + (a * sn).abs()], dim=1))
        return {"qt": (torch.cat(out), torch.cat(terms))}
    w, b, wo, bo = f("self_attn.in_proj_weight"), f("self_attn.in_proj_bias"), f("self_attn.out_proj.weight"), f("self_attn.out_proj.bias")
    wv = [w[2 * D + h * HD:2 * D + (h + 1) * HD] for h in range(H)]
    fw = torch.cat([w[:2 * D]] + [wo[:, h * HD:(h + 1) * HD] @ wv[h] for h in range(H)])
    tw = torch.cat([w[:2 * D].abs()] + [wo[:, h * HD:(h + 1) * HD].abs() @ wv[h].abs() for h in range(H)])
    fb = torch.cat([b[:2 * D], torch.zeros(H * D, dtype=b.dtype)])
    bof = bo + sum(wo[:, h * HD:(h + 1) * HD] @ b[2 * D + h * HD:2 * D + (h + 1) * HD] for h in range(H))
    tbo = bo.abs() + sum(wo[:, h * HD:(h + 1) * HD].abs() @ b[2 * D + h * HD:2 * D + (h + 1) * HD].abs() for h in range(H))
    return {"qkvf_w": (fw, tw), "qkvf_b": (fb, fb.abs()), "bo_f": (bof, tbo)}


@gpu
@pytest.mark.parametrize("rotary", ["absolute", "bucketed"])
@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
def test_folded_operands(eng, record_property, rotary, backend):
    """commit-time folds within one fp32 rounding of float64 (plus 2^-50 of the summed magnitudes for the double sums);
    bind-time memory tensors within the GEMM bounds composed through kv = cond Wkv^T + b, vp = V Wo_h^T, kp = K Wq_h / 8 and
    kc = (bq_h . K_h) / 8 (a 64-term fp32 warp sum: 7u of the summed magnitudes)"""
    from tests.helpers import mdm_weights
    sd = mdm_weights("smpl", "auto")
    eng.set_gemm_backend(backend)
    try:
        eng.load_denoiser(sd, "smpl", rotary=rotary)
        B, T, Tk = 3, 30, 10
        cond = torch.randn(Tk, B, D, generator=torch.Generator().manual_seed(8))
        eng.bind(cond, T)
        for layer in range(8):
            for name, (want, terms) in fold_reference(sd, layer, rotary).items():
                got = eng.denoiser_tensor(layer, name).cpu().double()
                bnd = U * want.abs() + 2.0 ** -50 * terms
                check(record_property, got.reshape(want.shape), want, bnd, "_%d_%s" % (layer, name))
            p = "decoder.layers.%d.multihead_attn." % layer
            w, b = torch.as_tensor(sd[p + "in_proj_weight"]).double().to(DEV), torch.as_tensor(sd[p + "in_proj_bias"]).double().to(DEV)
            wo = torch.as_tensor(sd[p + "out_proj.weight"]).double().to(DEV)
            X = cond.reshape(Tk * B, D).double().to(DEV)
            gb = (lambda A, W: simt_bound(A, W)) if backend == "simt" else (lambda A, W: tc_bound(A, W))
            kv = X @ w[D:].T + b[D:]
            ekv = gb(X, w[D:]) + U * kv.abs()
            kp, vp, kc = [], [], []
            ekp, evp, ekc = [], [], []
            for h in range(H):
                K, V = kv[:, h * HD:(h + 1) * HD], kv[:, D + h * HD:D + (h + 1) * HD]
                eK, eV = ekv[:, h * HD:(h + 1) * HD], ekv[:, D + h * HD:D + (h + 1) * HD]
                Wo, Wq = wo[:, h * HD:(h + 1) * HD], w[h * HD:(h + 1) * HD]
                vp.append(V @ Wo.T); evp.append(SLACK * (eV @ Wo.abs().T + gb(V, Wo)))
                kp.append(K @ Wq / 8); ekp.append(SLACK * (eK @ Wq.abs() + gb(K, Wq.T)) / 8)
                bq = b[h * HD:(h + 1) * HD]
                kc.append(K @ bq / 8); ekc.append(SLACK * (eK @ bq.abs() + 7 * U * (K.abs() @ bq.abs())) / 8)
            for name, want, e in (("kp", torch.cat(kp, 1), torch.cat(ekp, 1)), ("vp", torch.cat(vp, 1), torch.cat(evp, 1)),
                                  ("kc", torch.stack(kc, 1), torch.stack(ekc, 1))):
                check(record_property, eng.denoiser_tensor(layer, name), want, e, "_%d_%s" % (layer, name))
        from interdiff_b200.engine import EngineError
        with pytest.raises(EngineError, match="has no tensor"):
            eng.denoiser_tensor(0, "qt")
        with pytest.raises(EngineError, match="has no tensor"):
            eng.denoiser_tensor(1, "bo_f")
    finally:
        eng.set_gemm_backend("tcgen05")
