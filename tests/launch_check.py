"""Step-by-step checker of the engine's launch lists -- TEST INFRASTRUCTURE, never imported by the product.

``check_steps(steps, mem)`` runs a plan's steps (``_Plan.steps`` of Engine.plan / pair_plan / batch_plan, ``_TrackPlan.steps``)
in list order, one launch at a time on one stream, skipping fork / join: list order is a valid serialisation, because the
steps of one parallel branch keep their order.  For each step it

  1. takes float64 snapshots of everything the step reads (before the launch: upsample_add and groupnorm_relu work in place),
  2. launches the step and synchronises,
  3. compares every output the step wrote with a float64 restatement computed from the snapshots, element by element,
     against the bound below.

Memory is reached through the pointers of the argument lists (``Memory``): device memory through ``__cuda_array_interface__``,
host memory (the C-ABI emulation of tests/cabi_emulator.py) through ctypes buffers.  An entry point without a checker fails
the walk; the only steps run unchecked are the host-side ones listed in HOST_STEPS.

Bounds.  u = 2^-24 (fp32 unit roundoff); ulp_out(r) = spacing of the output dtype at r, subnormal floor included.

- conv (fp16 or fp32 storage, fp32 accumulation and epilogue), K = KH*KW*Cin, s / b = scale / bias of the output channel:
      |y - r| <= ulp_out(r) + 4u (K |s| sum|x w| + |b| + |res|)
  sum|x w| is the same convolution over |x| and |w|.  K u sum|x w| bounds a K-term fp32 dot product in any summation order
  (split-K partial sums included); the factor 4 allows for tensor-core fp32 accumulation that does not round to nearest
  and for the epilogue's roundings.  ReLU is 1-Lipschitz and keeps the bound.
- xcorr (NHWC and channel-planar windows): the same with K = T*T and no scale, bias or residual.
- upsample_add: ulp_out(r) + 8u (|lateral| + bilinear(|top|)): four products and four sums per element, exact weights
  (the pyramid levels differ by exactly 2x).
- roi_align, roi_align_planar, roi_align_batched: sample positions, cells and bilinear weights restated in fp32 exactly as
  the legacy ROIAlign specifies them, the samples summed in float64.  With cnt samples per bin,
      |y - r| <= ulp_out(r) + 2u (4 cnt + 2) S / cnt + 4u Q / cnt,
  S = sum over the samples of sum |w v| (fp32 accumulation of 4 cnt products), Q = sum over the samples of
  (|x| + |y| + 2) sum |v|: a sample position a few ulps off (a fused multiply-add where the restatement rounds twice) moves
  each bilinear weight by at most that much.
- deform_im2col3x3: each column element is one bilinear sample: ulp_out(r) + 4u sum|w v| + 4u (|x| + |y| + 2) sum|v|.
- groupnorm_relu (two passes in fp32 over the n = HW * C / groups values of a group): with m1 = mean |x| of the group,
  sigma = sqrt(var + eps) and z = (x - mean) / sigma in float64, in units of the normalised value z:
      |y - r| <= ulp_out(r) + 2 [ |g| ((n + 1) u m1 / sigma + (n / 2 + 8) u |z|) + 2u (|b| + |g z|) ]
  (n + 1) u m1 bounds the error of the fp32 mean (an n-term sum and a division), (n / 2 + 8) u the relative error of
  rsqrt(var + eps): half the n-term summation bound of the variance (the mean's error enters it only squared), rsqrtf's
  2 ulps and the subtraction; the last term is the affine epilogue.  Factor 2 of margin.
- maxpool2x2, maxpool3x3s2, subsample2: exact.  image_to_nhwc: exactly the fp32 image rounded to the storage dtype.
- rpn_select*, sort_nms*, box_decode*, track_combine*: the specification in cabi_emulator.FakeLib
  (batched_emulator.BatchedFakeLib) evaluated on host copies of the same fp32 inputs.  Counts, indices and labels exact,
  boxes within 1e-3 px, scores within 1e-6.
- emm_decode: FakeLib's restatement likewise: valid flags exact, boxes within 1e-3 px, confidences within 1e-5.  Where the
  reference's top-two margin on the response score is below 1e-5, either arg-max is accepted and the record notes it.
"""
import ctypes as C

import torch
import torch.nn.functional as F

U = 2.0 ** -24
F64 = torch.float64
BOX_BAR, SCORE_BAR, CONF_BAR = 1e-3, 1e-6, 1e-5

# host-side steps of the launch lists: run, not checked
HOST_STEPS = {"det_init": "host-side lambda of the plan: fills the detection block's scores with -1 and its count with 0 "
                          "(torch fill_ / zero_ on the plan's tensors; no libsmot entry point)"}

_DT = {0: torch.float32, 1: torch.float16}
_TYPESTR = {torch.float16: "<f2", torch.float32: "<f4", torch.int32: "<i4", torch.uint8: "|u1"}


def _addr(p):
    if p is None:
        return 0
    if isinstance(p, C.c_void_p):
        return p.value or 0
    return int(p)


def _contig(shape):
    st, acc = [], 1
    for n in reversed(shape):
        st.append(acc)
        acc *= n
    return tuple(reversed(st))


class _Cai(object):
    def __init__(self, ptr, shape, strides, dtype):
        item = torch.empty((), dtype=dtype).element_size()
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=_TYPESTR[dtype], data=(ptr, False),
                                             strides=tuple(s * item for s in strides), version=3)


class Memory(object):
    """Tensor views at raw addresses, over device memory ("cuda") or host memory ("cpu")."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"

    def view(self, ptr, shape, strides=None, dtype=torch.float32):
        shape = tuple(int(s) for s in shape)
        strides = _contig(shape) if strides is None else tuple(int(s) for s in strides)
        if any(n == 0 for n in shape):
            return torch.zeros(shape, dtype=dtype, device=self.device)
        ptr = _addr(ptr)
        assert ptr, "null operand pointer"
        if self.cuda:
            t = torch.as_tensor(_Cai(ptr, shape, strides, dtype), device=self.device)
            assert t.data_ptr() == ptr and t.stride() == strides
            return t
        item = torch.empty((), dtype=dtype).element_size()
        span = 1 + sum((n - 1) * s for n, s in zip(shape, strides))
        return torch.frombuffer((C.c_byte * (span * item)).from_address(ptr), dtype=dtype).as_strided(shape, strides)

    def nhwc(self, ptr, B, H, W, Cc, ld, dtype):
        return self.view(ptr, (B, H, W, Cc), (H * W * ld, W * ld, ld, 1), dtype)

    def rows(self, ptr, n, width, stride, dtype=torch.float32):
        return self.view(ptr, (n, width), (stride, 1), dtype)

    def host(self, ptr, shape, strides=None, dtype=torch.float32):
        """A contiguous host copy (fp32 / int32 inputs of the selection entry points)."""
        return self.view(ptr, shape, strides, dtype).cpu().contiguous().clone()


def ulp(r, dtype):
    """Spacing of `dtype` at |r| (subnormal floor included), float64."""
    mant, emin = (10, -14) if dtype == torch.float16 else (23, -126)
    e = torch.frexp(r.abs())[1].to(torch.int32) - 1                    # |r| in [2^e, 2^(e+1))
    e = torch.where(r == 0, torch.full_like(e, emin), torch.clamp(e, min=emin))
    return torch.ldexp(torch.ones_like(r, dtype=F64), (e - mant).to(F64))


class Check(object):
    """What one step's comparison found: worst |err| and worst |err| / bound (bound-checked outputs) or |err| / bar."""

    def __init__(self):
        self.max_err, self.max_ratio, self.where, self.notes = 0.0, 0.0, None, []

    def bound(self, what, y, r, bound):
        y, r = y.to(F64), r.to(F64)
        err = (y - r).abs()
        if err.numel() == 0:
            return
        ratio = err / bound
        bad = ~torch.isfinite(ratio)
        if bool(bad.any()):
            ratio = torch.where(bad, torch.full_like(ratio, float("inf")), ratio)
        k = int(torch.argmax(ratio))
        q = float(ratio.reshape(-1)[k])
        self.max_err = max(self.max_err, float(torch.where(bad, torch.zeros_like(err), err).max()))
        if q > self.max_ratio or self.where is None:
            idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), tuple(ratio.shape)))
            self.where = (what, idx, float(y.reshape(-1)[k]), float(r.reshape(-1)[k]), float(bound.reshape(-1)[k]))
            self.max_ratio = max(self.max_ratio, q)

    def bar(self, what, y, r, bar):
        y, r = y.to(F64).cpu(), r.to(F64).cpu()
        self.bound(what, y, r, torch.full_like(r, float(bar)))

    def exact(self, what, y, r):
        y, r = y.to(F64).cpu(), r.to(F64).cpu()
        if y.shape != r.shape:
            self.max_ratio, self.where = float("inf"), (what, "shape", tuple(y.shape), tuple(r.shape))
            return
        diff = (y != r) & ~(torch.isnan(y) & torch.isnan(r))
        if bool(diff.any()):
            k = int(diff.reshape(-1).nonzero()[0])
            self.max_err = max(self.max_err, float((y - r).abs().reshape(-1)[k]))
            self.max_ratio = float("inf")
            self.where = (what, tuple(int(i) for i in torch.unravel_index(torch.tensor(k), tuple(y.shape))),
                          float(y.reshape(-1)[k]), float(r.reshape(-1)[k]), 0.0)


# ------------------------------------------------------------------------------------------------------------------------
# dense kernels: float64 restatements with per-element bounds
# ------------------------------------------------------------------------------------------------------------------------
def conv_reference(x, w, d, scale, bias, res):
    """float64 reference and bound of smot_conv2d on snapshots x (B,H,W,Cin), w (Cout,KH,KW,Cin), fp32 scale / bias."""
    xc, wc = x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2)
    acc = F.conv2d(xc, wc, None, d.stride, d.pad)
    mag = F.conv2d(xc.abs(), wc.abs(), None, d.stride, d.pad)
    K = d.KH * d.KW * d.Cin
    s = scale.view(1, -1, 1, 1) if scale is not None else torch.ones((), dtype=F64, device=x.device)
    r = acc * s
    extra = torch.zeros((), dtype=F64, device=x.device)
    if bias is not None:
        r = r + bias.view(1, -1, 1, 1)
        extra = extra + bias.abs().view(1, -1, 1, 1)
    if res is not None:
        rr = res.permute(0, 3, 1, 2)
        r = r + rr
        extra = extra + rr.abs()
    if d.relu:
        r = r.clamp_min(0.0)
    r = r.permute(0, 2, 3, 1)
    b = (4 * U * (K * s.abs() * mag + extra)).permute(0, 2, 3, 1)
    return r, b + ulp(r, _DT[d.out_dtype])


def conv_snapshot(mem, d):
    idt = _DT[d.in_dtype]
    x = mem.nhwc(d.inp, d.batch, d.H, d.W, d.Cin, d.in_ld, idt).to(F64)
    w = mem.view(d.weight, (d.Cout, d.KH, d.KW, d.Cin), None, idt).to(F64)
    scale = mem.view(d.scale, (d.Cout,)).to(F64) if _addr(d.scale) else None
    bias = mem.view(d.bias, (d.Cout,)).to(F64) if _addr(d.bias) else None
    res = mem.nhwc(d.residual, d.batch, d.OH, d.OW, d.Cout, d.res_ld, idt).to(F64) if _addr(d.residual) else None
    return x, w, scale, bias, res


def check_conv(mem, d, launch):
    """Snapshot, launch(), compare: the conv part of the walker, usable on a descriptor built by hand."""
    snap = conv_snapshot(mem, d)
    launch()
    y = mem.nhwc(d.out, d.batch, d.OH, d.OW, d.Cout, d.out_ld, _DT[d.out_dtype])
    r, b = conv_reference(*snap[:2], d, *snap[2:])
    ck = Check()
    ck.bound("out", y, r, b)
    return ck


def _c_conv(ctx, args):
    return check_conv(ctx.mem, args[0]._obj, ctx.launch)


def _c_image(ctx, args):
    chw, out, Cc, H, W, ld, dt = args
    src = ctx.mem.view(chw, (Cc, H, W)).clone()
    ctx.launch()
    ck = Check()
    ck.exact("out", ctx.mem.nhwc(out, 1, H, W, Cc, ld, _DT[dt])[0], src.permute(1, 2, 0).to(_DT[dt]))
    return ck


def _c_pool(kind):
    def chk(ctx, args):
        inp, out, B, H, W, Cc, ild, old, dt = args
        x = ctx.mem.nhwc(inp, B, H, W, Cc, ild, _DT[dt]).to(F64).permute(0, 3, 1, 2)
        ctx.launch()
        r = F.max_pool2d(x, 2, 2) if kind == 2 else F.max_pool2d(x, 3, 2, 1)
        ck = Check()
        ck.exact("out", ctx.mem.nhwc(out, B, r.shape[2], r.shape[3], Cc, old, _DT[dt]), r.permute(0, 2, 3, 1))
        return ck
    return chk


def _c_subsample(ctx, args):
    inp, out, H, W, Cc, ild, old, dt = args
    r = ctx.mem.nhwc(inp, 1, H, W, Cc, ild, _DT[dt]).to(F64)[:, ::2, ::2]
    ctx.launch()
    ck = Check()
    ck.exact("out", ctx.mem.nhwc(out, 1, r.shape[1], r.shape[2], Cc, old, _DT[dt]), r)
    return ck


def _c_upsample_add(ctx, args):
    top, Ht, Wt, tld, lat, H, W, lld, Cc, dt = args
    t = ctx.mem.nhwc(top, 1, Ht, Wt, Cc, tld, _DT[dt]).to(F64).permute(0, 3, 1, 2)
    l0 = ctx.mem.nhwc(lat, 1, H, W, Cc, lld, _DT[dt]).to(F64)
    ctx.launch()
    up = F.interpolate(t, size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    upa = F.interpolate(t.abs(), size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    r = l0 + up
    ck = Check()
    ck.bound("lateral", ctx.mem.nhwc(lat, 1, H, W, Cc, lld, _DT[dt]), r, ulp(r, _DT[dt]) + 8 * U * (l0.abs() + upa))
    return ck


def _c_groupnorm(ctx, args):
    x, gamma, beta, batch, HW, Cc, ld, groups, eps, relu, dt = args
    v = ctx.mem.nhwc(x, batch, 1, HW, Cc, ld, _DT[dt]).to(F64)[:, 0]
    g = ctx.mem.view(gamma, (Cc,)).to(F64)
    b = ctx.mem.view(beta, (Cc,)).to(F64)
    ctx.launch()
    cpg = Cc // groups
    n = HW * cpg
    vg = v.reshape(batch, HW, groups, cpg)
    mean = vg.mean(dim=(1, 3), keepdim=True)
    var = ((vg - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    sigma = torch.sqrt(var + float(C.c_float(eps).value))
    z = (vg - mean) / sigma
    m1 = vg.abs().mean(dim=(1, 3), keepdim=True)
    gg, bb = g.view(1, 1, groups, cpg), b.view(1, 1, groups, cpg)
    r = z * gg + bb
    if relu:
        r = r.clamp_min(0.0)
    bound = 2 * (gg.abs() * ((n + 1) * U * m1 / sigma + (n / 2 + 8) * U * z.abs()) + 2 * U * (bb.abs() + (gg * z).abs()))
    r = r.reshape(batch, HW, Cc)
    bound = bound.reshape(batch, HW, Cc) + ulp(r, _DT[dt])
    ck = Check()
    ck.bound("x", ctx.mem.nhwc(x, batch, 1, HW, Cc, ld, _DT[dt])[:, 0], r, bound)
    return ck


def _bilinear_terms(feat, yy, xx, H, W):
    """feat (H,W,C) float64; fp32 sample positions yy, xx (any equal shape S).  DCN v1 bilinear sampling (zero outside the
    map): returns value, sum |w v| and sum |v| over the four corners, each (*S, C)."""
    inside = (yy > -1) & (yy < H) & (xx > -1) & (xx < W)
    y0, x0 = torch.floor(yy), torch.floor(xx)
    ly, lx = yy - y0, xx - x0
    one = torch.ones((), dtype=torch.float32, device=yy.device)
    val = mag = vab = 0.0
    for dy_, dx_, wgt in ((0, 0, (one - ly) * (one - lx)), (0, 1, (one - ly) * lx), (1, 0, ly * (one - lx)), (1, 1, ly * lx)):
        yi, xi = (y0 + dy_).long(), (x0 + dx_).long()
        ok = inside & (yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)
        v = feat[yi.clamp(0, H - 1), xi.clamp(0, W - 1)] * ok[..., None].to(F64)
        w = wgt.to(F64)[..., None]
        val = val + w * v
        mag = mag + (w * v).abs()
        vab = vab + v.abs()
    return val, mag, vab


def _c_deform(ctx, args):
    inp, off, cols, H, W, Cc, ild, oild, OH, OW, old, stride, dt = args
    x = ctx.mem.nhwc(inp, 1, H, W, Cc, ild, _DT[dt]).to(F64)[0]
    o = ctx.mem.nhwc(off, 1, OH, OW, 18, oild, torch.float32)[0].clone()
    ctx.launch()
    dev = x.device
    oy = (torch.arange(OH, device=dev) * stride - 1).view(OH, 1).float()
    ox = (torch.arange(OW, device=dev) * stride - 1).view(1, OW).float()
    y = ctx.mem.nhwc(cols, 1, OH, OW, 9 * Cc, old, _DT[dt])[0]
    ck = Check()
    for k in range(9):
        i, j = divmod(k, 3)
        yy, xx = (oy + i) + o[..., 2 * k], (ox + j) + o[..., 2 * k + 1]
        val, mag, vab = _bilinear_terms(x, yy, xx, H, W)
        pos = (yy.abs() + xx.abs() + 2).to(F64)[..., None]
        ck.bound("tap%d" % k, y[..., k * Cc:(k + 1) * Cc], val, ulp(val, _DT[dt]) + 4 * U * mag + 4 * U * pos * vab)
    return ck


def _roi_reference(mem, p, rois, lboxes, n, max_rois, Cc, res, sampling, dt, img=0, img_stride=None):
    """float64 ROIAlign (legacy, in-kernel level mapping, optional zero padding) of rows [0, n) and its bound; rows >= n are
    zero.  rois / lboxes: fp32 (max_rois, 4) tensors on the memory's device.  Snapshots the pyramid levels it reads."""
    dev = mem.device
    out = torch.zeros((max_rois, res, res, Cc), dtype=F64, device=dev)
    bnd = torch.zeros_like(out)
    if n == 0:
        return out, bnd
    assert sampling > 0
    lb = lboxes[:n]
    area = (lb[:, 2] - lb[:, 0] + 1) * (lb[:, 3] - lb[:, 1] + 1)
    lv = torch.floor(4 + torch.log2(torch.sqrt(area) / 224 + 1e-6))
    lv = lv.clamp(p.k_min, p.k_min + p.num_levels - 1).long() - p.k_min
    cnt = sampling * sampling
    ph = torch.arange(res, device=dev, dtype=torch.float32)
    it = torch.arange(sampling, device=dev, dtype=torch.float32) + 0.5
    for l in range(p.num_levels):
        idx = (lv == l).nonzero().squeeze(1)
        if idx.numel() == 0:
            continue
        H, W, ld, pad, sc = p.H[l], p.W[l], p.ld[l], p.pad[l], float(p.scale[l])
        base = _addr(p.feat[l]) + (img * int(img_stride[l]) * torch.empty((), dtype=_DT[dt]).element_size() if img else 0)
        feat = mem.nhwc(base, 1, H, W, Cc, ld, _DT[dt])[0].to(F64).reshape(H * W, Cc)
        Hp, Wp = H + 2 * pad, W + 2 * pad
        for chunk in idx.split(16):
            r = rois[chunk]
            sc32 = torch.tensor(sc, dtype=torch.float32, device=dev)
            x1, y1, x2, y2 = r[:, 0] * sc32, r[:, 1] * sc32, r[:, 2] * sc32, r[:, 3] * sc32
            rw, rh = (x2 - x1).clamp_min(1.0), (y2 - y1).clamp_min(1.0)
            bw, bh = rw / res, rh / res

            def pos(v1, bsz):   # (m, res * sampling) sample coordinates, fp32 as the legacy kernel forms them
                q = (it[None, :] * bsz[:, None]) / sampling
                return (v1[:, None, None] + ph[None, :, None] * bsz[:, None, None] + q[:, None, :]).reshape(len(v1), -1)

            def cell(v, Lp):
                ok = ~((v < -1) | (v > Lp))
                vv = torch.where(v <= 0, torch.zeros_like(v), v)
                lo = vv.long()
                top = lo >= Lp - 1
                lo = torch.where(top, torch.full_like(lo, Lp - 1), lo)
                hi = torch.where(top, lo, lo + 1)
                vv = torch.where(top, lo.float(), vv)
                lam = vv - lo.float()
                return ok, lo, hi, lam, 1 - lam

            ys, xs = pos(y1, bh), pos(x1, bw)
            oky, yl, yh, ly, hy = cell(ys, Hp)
            okx, xl, xh, lx, hx = cell(xs, Wp)
            m = len(chunk)
            val = torch.zeros((m, ys.shape[1], xs.shape[1], Cc), dtype=F64, device=dev)
            mag, vab = torch.zeros_like(val), torch.zeros_like(val)
            for (yi, wy), (xi, wx) in (((yl, hy), (xl, hx)), ((yl, hy), (xh, lx)), ((yh, ly), (xl, hx)), ((yh, ly), (xh, lx))):
                ry, rx = yi - pad, xi - pad
                ok = ((ry >= 0) & (ry < H))[:, :, None] & ((rx >= 0) & (rx < W))[:, None, :]
                ok = ok & oky[:, :, None] & okx[:, None, :]
                flat = ry.clamp(0, H - 1)[:, :, None] * W + rx.clamp(0, W - 1)[:, None, :]
                v = feat[flat] * ok[..., None].to(F64)
                w = (wy[:, :, None] * wx[:, None, :]).to(F64)[..., None]
                val += w * v
                mag += (w * v).abs()
                vab += v.abs()
            p_abs = (ys.abs()[:, :, None] + xs.abs()[:, None, :] + 2).to(F64)[..., None]
            shp = (m, res, sampling, res, sampling, Cc)
            tot = val.reshape(shp).sum(dim=(2, 4)) / cnt
            S = mag.reshape(shp).sum(dim=(2, 4))
            Q = (p_abs * vab).reshape(shp).sum(dim=(2, 4))
            out[chunk] = tot
            bnd[chunk] = 2 * U * (4 * cnt + 2) * S / cnt + 4 * U * Q / cnt
    return out, bnd + ulp(out, _DT[dt])


def _roi_inputs(mem, rois, level_boxes, count, max_rois):
    r = mem.view(rois, (max_rois, 4)).clone()
    lb = mem.view(level_boxes, (max_rois, 4)).clone() if _addr(level_boxes) else r
    n = max_rois if not _addr(count) else min(int(mem.view(count, (1,), None, torch.int32)[0]), max_rois)
    return r, lb, n


def _c_roi_align(ctx, args):
    pref, rois, level_boxes, count, max_rois, Cc, res, sampling, out, dt = args
    r, lb, n = _roi_inputs(ctx.mem, rois, level_boxes, count, max_rois)
    ref, bnd = _roi_reference(ctx.mem, pref._obj, r, lb, n, max_rois, Cc, res, sampling, dt)
    ctx.launch()
    ck = Check()
    ck.bound("out", ctx.mem.nhwc(out, max_rois, res, res, Cc, Cc, _DT[dt]), ref, bnd)
    return ck


def _c_roi_align_planar(ctx, args):
    pref, rois, level_boxes, count, max_rois, Cc, res, sampling, out, row_pitch, plane_pitch, dt = args
    r, lb, n = _roi_inputs(ctx.mem, rois, level_boxes, count, max_rois)
    ref, bnd = _roi_reference(ctx.mem, pref._obj, r, lb, n, max_rois, Cc, res, sampling, dt)
    ctx.launch()
    y = ctx.mem.view(out, (max_rois, res, res, Cc), (Cc * plane_pitch, row_pitch, 1, plane_pitch), _DT[dt])
    ck = Check()
    ck.bound("out", y, ref, bnd)
    return ck


def _c_roi_align_batched(ctx, args):
    pref, strides, batch, rois, count, max_rois, Cc, res, sampling, out, dt = args
    p = pref._obj
    refs = []
    for b in range(batch):
        r = ctx.mem.view(_addr(rois) + 16 * b * max_rois, (max_rois, 4)).clone()
        n = min(int(ctx.mem.view(_addr(count) + 4 * b, (1,), None, torch.int32)[0]), max_rois)
        refs.append(_roi_reference(ctx.mem, p, r, r, n, max_rois, Cc, res, sampling, dt, img=b, img_stride=strides))
    ctx.launch()
    ck = Check()
    y = ctx.mem.nhwc(out, batch * max_rois, res, res, Cc, Cc, _DT[dt])
    for b, (ref, bnd) in enumerate(refs):
        ck.bound("image%d" % b, y[b * max_rois:(b + 1) * max_rois], ref, bnd)
    return ck


def _xcorr_check(ctx, x, k, out_view_fn):
    """x (n,C,S,S), k (n,C,T,T) float64 snapshots."""
    ctx.launch()
    n, Cc, S = x.shape[0], x.shape[1], x.shape[2]
    T = k.shape[2]
    xs, ks = x.reshape(1, n * Cc, S, S), k.reshape(n * Cc, 1, T, T)
    r = F.conv2d(xs, ks, groups=n * Cc).reshape(n, Cc, S - T + 1, S - T + 1).permute(0, 2, 3, 1)
    a = F.conv2d(xs.abs(), ks.abs(), groups=n * Cc).reshape(n, Cc, S - T + 1, S - T + 1).permute(0, 2, 3, 1)
    ck = Check()
    ck.bound("out", out_view_fn(), r, ulp(r, ctx.xdt) + 4 * U * T * T * a)
    return ck


def _c_xcorr(ctx, args):
    x, k, out, n, Cc, S, T, dt = args
    ctx.xdt = _DT[dt]
    if n == 0:
        ctx.launch()
        return Check()
    xs = ctx.mem.nhwc(x, n, S, S, Cc, Cc, _DT[dt]).to(F64).permute(0, 3, 1, 2)
    ks = ctx.mem.nhwc(k, n, T, T, Cc, Cc, _DT[dt]).to(F64).permute(0, 3, 1, 2)
    O = S - T + 1
    return _xcorr_check(ctx, xs, ks, lambda: ctx.mem.nhwc(out, n, O, O, Cc, Cc, _DT[dt]))


def _c_xcorr_planar(ctx, args):
    from siammot_b200 import _lib
    xp, k, out, n, Cc = args[:5]
    ctx.xdt = torch.float16                    # the planar exchange is the fp16 correlation
    if n == 0:
        ctx.launch()
        return Check()
    S, T, O, RP, PL = 30, 15, 16, _lib.XCORR_ROW_PITCH, _lib.XCORR_PLANE
    xs = ctx.mem.view(xp, (n, Cc, S, S), (Cc * PL, PL, RP, 1), torch.float16).to(F64)
    pad_cols = ctx.mem.view(_addr(xp) + 2 * S, (n, Cc, S, 2), (Cc * PL, PL, RP, 1), torch.float16)
    assert float(pad_cols.abs().max()) == 0.0, "columns 30 / 31 of the planar windows must be zero"
    ks = ctx.mem.nhwc(k, n, T, T, Cc, Cc, torch.float16).to(F64).permute(0, 3, 1, 2)
    return _xcorr_check(ctx, xs, ks, lambda: ctx.mem.nhwc(out, n, O, O, Cc, Cc, torch.float16))


# ------------------------------------------------------------------------------------------------------------------------
# selection / post-processing: FakeLib's specification on host copies of the same fp32 inputs
# ------------------------------------------------------------------------------------------------------------------------
def _hp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _spec():
    import batched_emulator
    return batched_emulator.BatchedFakeLib()


def _rpn_levels_host(mem, levels, num_levels, batch=1, strides=None):
    """Host copies of the RPN heads (images back to back) and smot_rpn_level structs over them."""
    lv = (type(levels[0]) * num_levels)()
    keep, hstr = [], (C.c_longlong * num_levels)()
    for l in range(num_levels):
        L = levels[l]
        hw, w = L.H * L.W, 5 * L.A
        st = int(strides[l]) if strides is not None else hw * L.head_ld
        h = mem.host(L.head, (batch, hw, w), (st, L.head_ld, 1))
        keep.append(h)
        lv[l] = type(L).from_buffer_copy(L)
        lv[l].head, lv[l].head_ld = h.data_ptr(), w
        hstr[l] = hw * w
    return lv, hstr, keep


def _compare_props(ck, mem, out_boxes, out_scores, out_count, hb, hs, hc, fpn_n, batch):
    cnt = mem.host(out_count, (batch,), None, torch.int32)
    ck.exact("count", cnt, hc)
    yb = mem.host(out_boxes, (batch, fpn_n, 4))
    ys = mem.host(out_scores, (batch, fpn_n))
    for b in range(batch):
        k = int(hc[b])
        ck.bar("boxes", yb[b, :k], hb[b, :k], BOX_BAR)
        ck.bar("scores", ys[b, :k], hs[b, :k], SCORE_BAR)


def _c_rpn_select(ctx, args):
    (levels, num_levels, pre_n, post_n, nms, min_size, fpn_n, img_w, img_h, amodal, out_boxes, out_scores, out_count,
     ws, ws_bytes) = args
    lv, _, keep = _rpn_levels_host(ctx.mem, levels, num_levels)
    hb, hs, hc = torch.zeros((1, fpn_n, 4)), torch.zeros((1, fpn_n)), torch.zeros((1,), dtype=torch.int32)
    _spec().smot_rpn_select(lv, num_levels, pre_n, post_n, nms, min_size, fpn_n, img_w, img_h, amodal, _hp(hb), _hp(hs), _hp(hc),
                            None, 0, None)
    ctx.launch()
    ck = Check()
    _compare_props(ck, ctx.mem, out_boxes, out_scores, out_count, hb, hs, hc, fpn_n, 1)
    return ck


def _c_rpn_select_batched(ctx, args):
    (levels, strides, batch, num_levels, pre_n, post_n, nms, min_size, fpn_n, img_w, img_h, amodal, out_boxes, out_scores,
     out_count, ws, ws_bytes) = args
    lv, hstr, keep = _rpn_levels_host(ctx.mem, levels, num_levels, batch, strides)
    hb, hs = torch.zeros((batch, fpn_n, 4)), torch.zeros((batch, fpn_n))
    hc = torch.zeros((batch,), dtype=torch.int32)
    _spec().smot_rpn_select_batched(lv, hstr, batch, num_levels, pre_n, post_n, nms, min_size, fpn_n, img_w, img_h, amodal,
                                    _hp(hb), _hp(hs), _hp(hc), None, 0, None)
    ctx.launch()
    ck = Check()
    _compare_props(ck, ctx.mem, out_boxes, out_scores, out_count, hb, hs, hc, fpn_n, batch)
    return ck


def _c_sort_nms(ctx, args):
    (boxes, box_stride, scores, score_stride, count, n_max, min_score, thresh, max_keep, tag, out_index, out_boxes, out_scores,
     out_tag, out_count, ws, ws_bytes) = args
    m = ctx.mem
    base = int(m.view(out_count, (1,), None, torch.int32)[0])
    cap = base + min(max_keep, n_max)
    hb = m.host(boxes, (n_max, 4), (box_stride, 1))
    hs = m.host(scores, (n_max,), (score_stride,))
    hcount = m.host(count, (1,), None, torch.int32) if _addr(count) else None
    outs = dict(index=(out_index, torch.int32, (cap,)), boxes=(out_boxes, torch.float32, (cap, 4)),
                scores=(out_scores, torch.float32, (cap,)), tag=(out_tag, torch.int32, (cap,)))
    host = {k: torch.zeros(shape, dtype=dt) if _addr(p) else None for k, (p, dt, shape) in outs.items()}
    hc = torch.tensor([base], dtype=torch.int32)
    _spec().smot_sort_nms(_hp(hb), 4, _hp(hs), 1, _hp(hcount), n_max, min_score, thresh, max_keep, tag, _hp(host["index"]),
                          _hp(host["boxes"]), _hp(host["scores"]), _hp(host["tag"]), _hp(hc), None, 0, None)
    ctx.launch()
    ck = Check()
    got = int(m.view(out_count, (1,), None, torch.int32)[0])
    ck.exact("count", torch.tensor([got]), hc)
    k = int(hc[0])
    if got == k and k > base:
        for name, (p, dt, shape) in outs.items():
            if host[name] is None:
                continue
            y = m.host(p, shape, None, dt)[base:k]
            if name == "boxes":
                ck.bar(name, y, host[name][base:k], BOX_BAR)
            elif name == "scores":
                ck.bar(name, y, host[name][base:k], SCORE_BAR)
            else:
                ck.exact(name, y, host[name][base:k])
    return ck


def _c_sort_nms_segmented(ctx, args):
    (boxes, scores, count, batch, n_max, ncls, min_score, thresh, max_keep, cap, out_boxes, out_scores, out_block, ws,
     ws_bytes) = args
    m = ctx.mem
    hb = m.host(boxes, (batch * n_max * ncls * 4,))
    hs = m.host(scores, (batch * n_max * ncls,))
    hcount = m.host(count, (batch,), None, torch.int32)
    ob, os_ = torch.zeros((batch, cap, 4)), torch.zeros((batch, cap))
    blk = torch.zeros((batch, 1 + cap), dtype=torch.int32)
    _spec().smot_sort_nms_segmented(_hp(hb), _hp(hs), _hp(hcount), batch, n_max, ncls, min_score, thresh, max_keep, cap, _hp(ob),
                                    _hp(os_), _hp(blk), None, 0, None)
    ctx.launch()
    ck = Check()
    yblk = m.host(out_block, (batch, 1 + cap), None, torch.int32)
    ck.exact("count", yblk[:, 0], blk[:, 0])
    ys = m.host(out_scores, (batch, cap))
    yb = m.host(out_boxes, (batch, cap, 4))
    for b in range(batch):
        k = int(blk[b, 0])
        if int(yblk[b, 0]) != k:
            continue
        ck.exact("labels", yblk[b, 1:1 + k], blk[b, 1:1 + k])
        ck.bar("scores", ys[b], os_[b], SCORE_BAR)
        ck.bar("boxes", yb[b, :k], ob[b, :k], BOX_BAR)
    return ck


def _c_box_decode(ctx, args):
    head, head_ld, rois, count, n_max, ncls, w4ref, img_w, img_h, amodal, track_labels, out_boxes, out_scores = args
    m = ctx.mem
    hh = m.host(head, (n_max, 5 * ncls), (head_ld, 1))
    hr = m.host(rois, (n_max, 4))
    hcount = m.host(count, (1,), None, torch.int32) if _addr(count) else None
    hl = m.host(track_labels, (n_max,), None, torch.int32) if _addr(track_labels) else None
    ob, os_ = torch.zeros((n_max, 4 * ncls)), torch.zeros((n_max, ncls))
    _spec().smot_box_decode(_hp(hh), 5 * ncls, _hp(hr), _hp(hcount), n_max, ncls, w4ref, img_w, img_h, amodal, _hp(hl), _hp(ob),
                            _hp(os_), None)
    ctx.launch()
    ck = Check()
    ck.bar("boxes", m.host(out_boxes, (n_max, 4 * ncls)), ob, BOX_BAR)
    ck.bar("scores", m.host(out_scores, (n_max, ncls)), os_, SCORE_BAR)
    return ck


def _c_box_decode_batched(ctx, args):
    head, head_ld, rois, count, batch, n_max, ncls, w4ref, img_w, img_h, amodal, out_boxes, out_scores = args
    m = ctx.mem
    hh = m.host(head, (batch * n_max, 5 * ncls), (head_ld, 1))
    hr = m.host(rois, (batch * n_max, 4))
    hcount = m.host(count, (batch,), None, torch.int32)
    ob, os_ = torch.zeros((batch * n_max, 4 * ncls)), torch.zeros((batch * n_max, ncls))
    _spec().smot_box_decode_batched(_hp(hh), 5 * ncls, _hp(hr), _hp(hcount), batch, n_max, ncls, w4ref, img_w, img_h, amodal,
                                    _hp(ob), _hp(os_), None)
    ctx.launch()
    ck = Check()
    ck.bar("boxes", m.host(out_boxes, (batch * n_max, 4 * ncls)), ob, BOX_BAR)
    ck.bar("scores", m.host(out_scores, (batch * n_max, ncls)), os_, SCORE_BAR)
    return ck


def _combine(grouped):
    def chk(ctx, args):
        m = ctx.mem
        (det_boxes, det_scores, ncap, dec_boxes, dec_scores, ncls, labels, conf, valid, active, n, tracktor, cat_boxes,
         cat_scores, zero_count) = args[:15]
        perm = args[15] if grouped else None
        hd = [m.host(det_boxes, (ncap, 4)), m.host(det_scores, (ncap,))]
        if n:
            hn = [m.host(dec_boxes, (n, 4 * ncls)), m.host(dec_scores, (n, ncls)), m.host(labels, (n,), None, torch.int32),
                  m.host(conf, (n,)), m.host(valid, (n,), None, torch.int32), m.host(active, (n,))]
        else:
            hn = [None] * 6
        cb, cs = torch.zeros((ncap + n, 4)), torch.zeros((ncap + n,))
        zc = torch.full((1,), 7, dtype=torch.int32) if _addr(zero_count) else None
        hp = torch.zeros((n,), dtype=torch.int32) if grouped else None
        a = [_hp(hd[0]), _hp(hd[1]), ncap, _hp(hn[0]), _hp(hn[1]), ncls] + [_hp(t) for t in hn[2:]] + [n, tracktor, _hp(cb),
                                                                                                      _hp(cs), _hp(zc)]
        spec = _spec()
        if grouped:
            spec.smot_track_combine_grouped(*a, _hp(hp), None)
        else:
            spec.smot_track_combine(*a, None)
        ctx.launch()
        ck = Check()
        ck.bar("cat_boxes", m.host(cat_boxes, (ncap + n, 4)), cb, BOX_BAR)
        ck.bar("cat_scores", m.host(cat_scores, (ncap + n,)), cs, SCORE_BAR)
        if zc is not None:
            ck.exact("zero_count", m.host(zero_count, (1,), None, torch.int32), zc)
        if grouped and n:
            ck.exact("perm", m.host(perm, (n,), None, torch.int32), hp)
        return ck
    return chk


def _emm_scores(maps, sr, tb, pad, T, use_ctr, sigma, up):
    """oracle.siammot_oracle.emm_decode's score map and per-location terms (fp32, host): for the top-two margin."""
    cls, ctr, reg = maps[:, 0:2], maps[:, 2:3], maps[:, 3:7]
    n = cls.shape[0]
    cls_u = F.interpolate(cls, scale_factor=up, mode="bicubic")
    ctr_u = F.interpolate(ctr, scale_factor=up, mode="bicubic")
    reg_u = F.interpolate(reg, scale_factor=up, mode="bicubic")
    p1 = F.softmax(cls_u, dim=1)[:, 1].reshape(n, -1)
    conf = p1 * torch.sigmoid(ctr_u).reshape(n, -1) if use_ctr else p1
    tlbr = reg_u.reshape(n, 4, -1)
    sw = (tlbr[:, 2] + tlbr[:, 0]) / (tb[:, 2] - tb[:, 0])[:, None]
    sh = (tlbr[:, 3] + tlbr[:, 1]) / (tb[:, 3] - tb[:, 1])[:, None]
    sw, sh = torch.max(sw, 1 / sw), torch.max(sh, 1 / sh)
    side = cls_u.shape[-1]
    hann = torch.hann_window(side, dtype=torch.float)
    score = (conf * torch.exp((-sw * sh + 1) * 0.1)) * (1 - sigma) + sigma * torch.outer(hann, hann).reshape(-1)[None]
    return score, p1, tlbr, side


def _c_emm_decode(ctx, args):
    from oracle import prims
    (maps, map_ld, n, O, up, T, sr, tboxes, hann, pad, use_ctr, sigma, img_w, img_h, amodal, out_boxes, out_conf, out_valid,
     scratch) = args
    m = ctx.mem
    if n == 0:
        ctx.launch()
        return Check()
    hm = m.host(maps, (n, O, O, 7), (O * O * map_ld, O * map_ld, map_ld, 1))
    hs, ht = m.host(sr, (n, 4)), m.host(tboxes, (n, 4))
    hh = m.host(hann, (O * up,))
    ob, oc, ov = torch.zeros((n, 4)), torch.zeros((n,)), torch.zeros((n,), dtype=torch.int32)
    _spec().smot_emm_decode(_hp(hm), 7, n, O, up, T, _hp(hs), _hp(ht), _hp(hh), pad, use_ctr, sigma, img_w, img_h, amodal, _hp(ob),
                            _hp(oc), _hp(ov), None, None)
    ctx.launch()
    yb, yc, yv = m.host(out_boxes, (n, 4)), m.host(out_conf, (n,)), m.host(out_valid, (n,), None, torch.int32)
    ck = Check()
    row_bad = ((yb - ob).abs().amax(1) > BOX_BAR) | ((yc - oc).abs() > CONF_BAR) | (yv != ov)
    if bool(row_bad.any()):
        # a near-tie of the reference's arg-max: accept the runner-up location when the margin is below the fp32 bar
        score, p1, tlbr, side = _emm_scores(hm.permute(0, 3, 1, 2), hs, ht, pad, T, use_ctr, float(sigma), up)
        top = torch.topk(score, 2, dim=1)
        s_full = (O + 2 * (T // 2)) * up
        border = (T // 2) * up
        ar = torch.arange(0, s_full, dtype=torch.float32)
        for r in row_bad.nonzero().squeeze(1).tolist():
            if float(top.values[r, 0] - top.values[r, 1]) > CONF_BAR:
                continue
            idx = int(top.indices[r, 1])
            bw, bh = hs[r, 2] - hs[r, 0], hs[r, 3] - hs[r, 1]
            cx = (hs[r, 0] + ar * (bw / (s_full - 1)))[border:-border][idx % side] - pad
            cy = (hs[r, 1] + ar * (bh / (s_full - 1)))[border:-border][idx // side] - pad
            d = tlbr[r, :, idx]
            bb = torch.stack((cx - d[0], cy - d[1], cx + d[2], cy + d[3]))[None]
            valid = torch.ones(1, dtype=torch.int32)
            if not amodal:
                bb = prims.clip_boxes(bb, img_w, img_h)
                valid = prims.nonempty_mask(bb).to(torch.int32)
            ob[r], oc[r], ov[r] = bb[0], p1[r, idx], valid[0]
            ck.notes.append("emm_decode row %d: reference top-two margin %.2e, runner-up arg-max accepted"
                            % (r, float(top.values[r, 0] - top.values[r, 1])))
    ck.exact("valid", yv, ov)
    ck.bar("boxes", yb, ob, BOX_BAR)
    ck.bar("conf", yc, oc, CONF_BAR)
    return ck


CHECKERS = {
    "smot_image_to_nhwc": _c_image, "smot_conv2d": _c_conv, "smot_maxpool2x2": _c_pool(2), "smot_maxpool3x3s2": _c_pool(3),
    "smot_subsample2": _c_subsample, "smot_upsample_add": _c_upsample_add, "smot_groupnorm_relu": _c_groupnorm,
    "smot_deform_im2col3x3": _c_deform, "smot_roi_align": _c_roi_align, "smot_roi_align_planar": _c_roi_align_planar,
    "smot_roi_align_batched": _c_roi_align_batched, "smot_xcorr": _c_xcorr, "smot_xcorr_planar_mode": _c_xcorr_planar,
    "smot_emm_decode": _c_emm_decode, "smot_rpn_select": _c_rpn_select, "smot_rpn_select_batched": _c_rpn_select_batched,
    "smot_sort_nms": _c_sort_nms, "smot_sort_nms_segmented": _c_sort_nms_segmented, "smot_box_decode": _c_box_decode,
    "smot_box_decode_batched": _c_box_decode_batched, "smot_track_combine": _combine(False),
    "smot_track_combine_grouped": _combine(True),
}


class _Ctx(object):
    def __init__(self, mem, fn, args, tag):
        self.mem, self.fn, self.args, self.tag = mem, fn, args, tag
        self.xdt = None

    def launch(self):
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream) if self.mem.cuda else C.c_void_p(0)
        rc = self.fn(*self.args, st)
        if self.mem.cuda:
            torch.cuda.synchronize()
        if rc != 0:
            from siammot_b200 import _lib
            raise AssertionError("step %s failed (code %d): %s" % (self.tag, rc, _lib.lib().smot_last_error()))


def describe_conv(d):
    return ("b%d %dx%dx%d->%dx%dx%d k%dx%d s%d in_ld %d out_ld %d res_ld %d %s->%s"
            % (d.batch, d.H, d.W, d.Cin, d.OH, d.OW, d.Cout, d.KH, d.KW, d.stride, d.in_ld, d.out_ld, d.res_ld,
               "f16" if d.in_dtype else "f32", "f16" if d.out_dtype else "f32"))


def check_steps(steps, mem, lib=None, strict=True):
    """Run and check every step of a launch list in order (see the module docstring).  Returns one record per non-fork/join
    step: dict(step, tag, entry, conv, algo, checked, max_err, max_ratio, where, notes).  strict: raise AssertionError after
    the walk when a step exceeded its bound / bar."""
    recs = []
    for i, st in enumerate(steps):
        fn, args, tag = st[0], st[1], st[2]
        if isinstance(fn, str) and fn in ("fork", "join"):
            continue
        name = getattr(fn, "__name__", None)
        rec = dict(step=i, tag=tag, entry=name, conv=None, algo=None, checked=False, max_err=0.0, max_ratio=0.0, where=None,
                   notes=[])
        if name not in CHECKERS:
            if tag in HOST_STEPS:
                fn(*args, C.c_void_p(0))
                rec["notes"].append(HOST_STEPS[tag])
                recs.append(rec)
                continue
            raise AssertionError("step %d (%s): entry point %r has no checker" % (i, tag, name))
        if name == "smot_conv2d":
            rec["conv"] = describe_conv(args[0]._obj)
            if lib is not None:
                rec["algo"] = int(lib.smot_conv2d_algo(args[0]))
        ck = CHECKERS[name](_Ctx(mem, fn, args, tag), args)
        rec.update(checked=True, max_err=ck.max_err, max_ratio=ck.max_ratio, where=ck.where, notes=ck.notes)
        recs.append(rec)
    if strict:
        bad = [r for r in recs if r["checked"] and not r["max_ratio"] <= 1.0]
        assert not bad, "steps over their bound:\n" + "\n".join(format_record(r) for r in bad)
    return recs


def format_record(r):
    s = "%3d %-22s %-28s |err| %.3e  ratio %.3f" % (r["step"], r["tag"], r["entry"], r["max_err"], r["max_ratio"])
    if r["conv"]:
        s += "  [%s algo %s]" % (r["conv"], r["algo"])
    if r["max_ratio"] > 1.0 and r["where"] is not None:
        s += "  worst at %s" % (r["where"],)
    for n in r["notes"]:
        s += "\n      note: " + n
    return s


def report(name, steps, recs):
    """Summary line + one line per record; also the count the walk is expected to reach."""
    listed = [st for st in steps if not (isinstance(st[0], str) and st[0] in ("fork", "join"))]
    host = [st for st in listed if st[2] in HOST_STEPS and getattr(st[0], "__name__", None) not in CHECKERS]
    checked = [r for r in recs if r["checked"]]
    worst = max(checked, key=lambda r: r["max_ratio"]) if checked else None
    head = ("%s: %d of %d listed steps checked (%d host-side), entry points %s; worst |err|/bound %.3f at step %d %s"
            % (name, len(checked), len(listed), len(host), sorted({r["entry"] for r in checked}),
               worst["max_ratio"] if worst else 0.0, worst["step"] if worst else -1, worst["tag"] if worst else "-"))
    return head, len(listed) - len(host), "\n".join([head] + [format_record(r) for r in recs])
