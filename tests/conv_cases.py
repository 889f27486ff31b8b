"""Edge cases of smot_conv2d and the harness that runs them -- TEST INFRASTRUCTURE, not a test module.

Every case is one convolution descriptor placed on a branch of the routing code (capi.cu, conv_tc.cu, conv_hires.cu,
conv_smalln.cu, conv_simt.cu): its shape, stride, dtypes, pitches and channel offsets, scale / bias / residual / ReLU, the
split-K workspace, the environment it needs, the kernels it must launch and a short reason naming the branch.  The
kernel expectations (names, split factor, small-N K slicing) are written for an H100 SXM with 132 SMs; the cases stay away
from the `grid <= sm_count` and `ntiles >= sm_count` boundaries, so they hold on any SM count from 120 to 144.

`run_case(case, pattern, mem, launch)` places the operands inside larger buffers -- a channel offset, a pixel pitch wider
than the channel count, MARGIN elements before and after -- fills every byte outside the operands with a NaN pattern and,
for workspace cases, the reserved SMOT_CONV_WS_COUNTER_BYTES of the workspace with a byte pattern, then launches and checks:

- the output against launch_check.conv_reference (the float64 restatement and per-element bound shared with the plan
  walker, tests/launch_check.py): within the bound for the "gauss" pattern, bit for bit for the "exact" pattern;
- that the margins and pitch gaps of the output, the whole input and residual buffers and the reserved workspace bytes
  are unchanged, bit for bit.

Exact pattern: small integers, mostly zero, with nonzeros placed on purpose -- the last row and column of each image, the
first and last channel of every 64-channel K chunk (so every K chunk of every split range contributes), the last tap --
a power-of-two scale and an integer bias and residual.  The generator asserts sum|x w| < 2^11 and
|s| sum|x w| + |b| + |res| < 2^10 at every output, so every fp32 partial sum in any order is an integer held exactly, and
every result is a multiple of 1/2 that the output dtype holds exactly: any dropped, doubled or misplaced product is an
integer error against a zero tolerance.
"""
import ctypes as C
import json
import os
import re
import zlib
import tempfile

import torch
import torch.nn.functional as F

import launch_check as lc

F16, F32 = torch.float16, torch.float32
DT = {"f16": F16, "f32": F32}
CODE = {F32: 0, F16: 1}
MARGIN = 64                                 # elements before and after every operand buffer
WS_COUNTER = 65536                          # SMOT_CONV_WS_COUNTER_BYTES
WS_DEFAULT = 48 << 20                       # ops.conv_workspace's size
NAN_BITS = {F16: 0x7D5A, F32: 0x7FC5A5A5}  # quiet NaNs with a payload: a kernel never produces them
WS_BYTE = 0xA5
SM_COUNT = 132                              # the SM count the expectations are written for (H100 SXM)


class Case(object):
    def __init__(self, name, family, why, B, H, W, Cin, Cout, k, kernels, stride=1, pad=None, dt="f16", odt=None,
                 in_ld=None, in_off=None, out_ld=None, out_off=None, res=False, res_ld=None, res_off=None, relu=True,
                 ws=None, env=None, splits=None, wk=None, in_fill="nan", algo=None, child_env=None):
        self.name, self.family, self.why = name, family, why
        self.B, self.H, self.W, self.Cin, self.Cout, self.k, self.stride = B, H, W, Cin, Cout, k, stride
        self.pad = k // 2 if pad is None else pad
        self.OH = (H + 2 * self.pad - k) // stride + 1
        self.OW = (W + 2 * self.pad - k) // stride + 1
        self.dt, self.odt = DT[dt], DT[odt or dt]
        al = 8 if self.dt == F16 else 4    # 16 bytes
        self.in_off = al if in_off is None else in_off
        self.in_ld = Cin + 2 * al if in_ld is None else in_ld
        ao = 8 if self.odt == F16 else 4
        self.out_off = ao if out_off is None else out_off
        self.out_ld = Cout + 2 * ao if out_ld is None else out_ld
        self.res = res
        self.res_off = al if res_off is None else res_off
        self.res_ld = (Cout + 2 * al if res_ld is None else res_ld) if res else 0
        self.relu = relu
        self.ws = WS_DEFAULT if ws == "default" else ws
        self.env = dict(env or {})
        self.child_env = dict(child_env or {})     # switches read once per process: run in a child process
        self.kernels = tuple(kernels)
        self.splits, self.wk = splits, wk
        self.in_fill = in_fill
        self.algo = algo if algo is not None else (2 if kernels and kernels[0].startswith("conv_tc_kernel") else 1)
        assert self.in_ld >= self.in_off + Cin and self.out_ld >= self.out_off + Cout
        assert not res or self.res_ld >= self.res_off + Cout

    @property
    def K(self):
        return self.k * self.k * self.Cin

    def macs(self):
        return self.B * self.OH * self.OW * self.Cout * self.K

    def __repr__(self):
        return self.name


# ------------------------------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------------------------------
def _tc(name, why, B, H, W, Cin, Cout, k, kern, splits=1, **kw):
    ks = ["conv_tc_kernel<%d,%d>" % kern] + (["splitk_reduce_kernel"] if splits > 1 and "SMOT_TC_SLICED" not in
                                             kw.get("env", {}) else [])
    return Case(name, "wgmma", why, B, H, W, Cin, Cout, k, ks, splits=splits, **kw)


def _ring_cases():
    """K chunks 1, 2, ring-1, ring, ring+1 and >= 2 passes round the ring, for each of the 8 <BN, STAGES> variants, at
    depths forced by SMOT_TC_STAGES (read on every call).  1x1 convs with Cin = 64 x chunks (3x3 Cin 64 for 9 chunks), on
    maps with ragged OH and OW (45 = 5 x 8 + 5, 120 = 7 x 16 + 8; 30 = 3 x 8 + 6)."""
    out = []
    # BN 256: Cout 512 over 48 tiles (48 x 2 = 96 >= min_ctas);  BN 128: Cout 384 over 32 tiles (32 x 3 = 96, never 256);
    # BN 64: Cout 64 over 32 tiles
    geo = {256: (45, 120, 512), 128: (30, 120, 384), 64: (30, 120, 64)}
    for bn, st, force, chunks in ((256, 3, "3", (1, 2, 3, 4, 7)), (256, 4, "4", (1, 2, 3, 4, 5, 9)),
                                  (128, 2, "2", (1, 2, 3, 5)), (128, 3, "3", (1, 2, 3, 4, 7)),
                                  (128, 6, "6", (1, 2, 5, 6, 7, 13)),
                                  (64, 2, "2", (1, 2, 3, 5)), (64, 4, "4", (1, 2, 3, 4, 5, 9)),
                                  (64, 8, "8", (1, 2, 7, 8, 9, 17))):
        H, W, cout = geo[bn]
        for c in chunks:
            k, cin = (3, 64) if c == 9 else (1, 64 * c)
            out.append(_tc("ring-bn%d-st%d-k%d" % (bn, st, c),
                           "tc_stages: SMOT_TC_STAGES=%s gives the %d-deep ring at BN %d; %d K chunk(s)" % (force, st, bn, c),
                           1, H, W, cin, cout, k, (bn, st), env={"SMOT_TC_STAGES": force}))
    return out


def _wgmma_cases():
    c = _ring_cases()
    c += [
        # ---- BN choice at min_ctas = 96
        _tc("bn-95-tiles", "BN: 95 tiles x Cout 128 / 128 = 95 < 96 keeps BN 64; 190 CTAs, not solo", 1, 40, 304, 64, 128, 1,
            (64, 4)),
        _tc("bn-96-tiles", "BN: 96 tiles x 128 / 128 = 96 takes BN 128; 96 CTAs solo, 1 chunk", 1, 64, 192, 64, 128, 1, (128, 3)),
        _tc("cout192-shallow", "BN 64 only (192 % 128 != 0); 100 tiles x 3 = 300 >= 296 and 1 chunk: shallow 2-stage ring",
            1, 80, 160, 64, 192, 1, (64, 2)),
        _tc("cout320-deep", "BN 64 only (320 % 128 != 0); 9 tiles x 5 CTAs solo, 9 chunks >= 6: 8-deep ring", 1, 22, 40, 64,
            320, 3, (64, 8)),
        _tc("cout384-bn128", "Cout 384: 32 tiles x 3 = 96 takes BN 128 (384 % 256 != 0: never 256)", 1, 30, 120, 128, 384, 1,
            (128, 3)),
        _tc("cout384-bn64", "Cout 384: 31 tiles x 3 = 93 < 96 keeps BN 64; 186 CTAs", 1, 8, 496, 128, 384, 1, (64, 4)),
        _tc("bn256-solo-deep", "BN 256 (96 tiles), 96 CTAs solo, 36 chunks >= 4: 4-deep", 1, 64, 192, 256, 256, 3, (256, 4)),
        _tc("bn256-crowded", "BN 256 (96 tiles x 2), 192 CTAs not solo: 3-deep", 1, 64, 192, 64, 512, 1, (256, 3)),
        # ---- feature-map tiles
        _tc("tile-tiny", "one 16x8 tile over a 5x9 map (OH < 8, OW < 16)", 1, 5, 9, 64, 64, 3, (64, 8)),
        _tc("tile-ragged-batch", "OH 21 = 2x8 + 5, OW 37 = 2x16 + 5, batch 2, residual with its own pitch (160, output 144)",
            2, 21, 37, 64, 128, 3, (64, 8), res=True, res_ld=160),
        _tc("route-m16", "batch*OH*OW = 16: the smallest map the wgmma route takes", 1, 4, 4, 64, 64, 3, (64, 8)),
        # ---- the H == 1 matrix path (128 x 1 tiles)
        _tc("rows-16", "H == 1: 128x1 tiles, 16 rows", 1, 1, 16, 256, 256, 1, (64, 4)),
        _tc("rows-127", "H == 1: 127 rows, one ragged tile", 1, 1, 127, 256, 256, 1, (64, 4)),
        _tc("rows-128", "H == 1: 128 rows, one full tile", 1, 1, 128, 256, 256, 1, (64, 4)),
        _tc("rows-129", "H == 1: 129 rows, a second tile of one row", 1, 1, 129, 256, 256, 1, (64, 4)),
        _tc("rows-300", "H == 1: 300 rows, 3 tiles", 1, 1, 300, 256, 256, 1, (64, 4)),
        _tc("rows-300-3x3", "H == 1 with a 3x3 filter: the rows above and below are TMA zero fill", 1, 1, 300, 64, 64, 3,
            (64, 8)),
        # ---- stride 2 (TMA element stride 2)
        _tc("s2-ow-odd", "stride 2, OW = 15 odd", 1, 20, 30, 64, 64, 3, (64, 8), stride=2),
        _tc("s2-batch-straddle", "stride 2, batch 3 of 6x10 outputs: the 16x8 tile's box runs past each image's bottom and "
            "right edge", 3, 12, 20, 64, 64, 3, (64, 8), stride=2),
        _tc("s2-split", "stride 2 with split-K: 4 tiles, 36 chunks -> 8 ranges of 5, the last of 1", 1, 22, 40, 256, 256, 3,
            (256, 4), stride=2, splits=8, ws="default"),
        # ---- pitches and alignment the route accepts
        _tc("ld-8mod64", "in_ld = 72, out_ld = 72 (8 mod 64): accepted (TMA strides are multiples of 16 bytes)", 1, 16, 32,
            64, 64, 3, (64, 8), in_ld=72, out_ld=72, in_off=8, out_off=0),
        # ---- split-K: the default rule (sp = min(148 / (tiles x Cout / BN), 8, chunks / 4)), ragged and rounded ranges
        _tc("split-3", "split 3: 39 tiles, 18 chunks -> 3 x 6; 117 CTAs solo, 6 chunks each: 8-deep", 1, 24, 208, 128, 64, 3,
            (64, 8), splits=3, ws="default"),
        _tc("split-4-ragged", "split 4: 30 tiles, 18 chunks -> 5, 5, 5, 3", 1, 24, 160, 128, 64, 3, (64, 4), splits=4,
            ws="default"),
        _tc("split-5-ragged", "split 5: 29 tiles, 27 chunks -> 6, 6, 6, 6, 3; 145 CTAs", 1, 8, 464, 192, 64, 3, (64, 4),
            splits=5, ws="default"),
        _tc("split-6-ragged", "split 6: 24 tiles, 27 chunks -> 5 x 5 + 2", 1, 24, 128, 192, 64, 3, (64, 4), splits=6,
            ws="default"),
        _tc("split-7", "split 7: 20 tiles, 28 chunks -> 7 x 4", 1, 32, 80, 1792, 64, 1, (64, 4), splits=7, ws="default"),
        _tc("split-8-level5", "split 8 at the level-5 shape (22x40x512 -> 128): 72 chunks -> 8 x 9, BN 128, 6-deep", 1, 22,
            40, 512, 128, 3, (128, 6), splits=8, ws="default"),
        _tc("split-empty-rounding", "33 chunks: 8 ranges of 5 would leave one empty, so 7 splits (6 x 5 + 3)", 1, 22, 40,
            2112, 64, 1, (64, 4), splits=7, ws="default"),
        _tc("split-ws-1-short", "the level-5 split-8 shape with a workspace one byte too small: no split, BN 64, 8-deep",
            1, 22, 40, 512, 128, 3, (64, 8), ws=WS_COUNTER + 8 * 9 * 128 * 128 * 4 - 1),
        _tc("split-batch10-2stage", "batch 10 of 3x3 256 -> 64 at 44x80: split 4 per image, 300 tiles x 1 >= 296 and 36 "
            "chunks: the 2-stage kernel with the reduce kernel", 10, 44, 80, 256, 64, 3, (64, 2), splits=4, ws="default"),
        _tc("fc6-30", "fc6 (K = 6272) at 30 rows: 1 tile, BN 256, split 8 (98 chunks -> 7 x 13 + 7)", 1, 1, 30, 6272, 1024,
            1, (256, 4), splits=8, ws="default", relu=True),
        _tc("fc6-300", "fc6 at 300 rows: 3 tiles x 4, split 8, 96 CTAs solo", 1, 1, 300, 6272, 1024, 1, (256, 4), splits=8,
            ws="default"),
        # ---- in-CTA K slices (SMOT_TC_SLICED, read on every call): the split ranges summed in one CTA
        _tc("sliced-level5", "SMOT_TC_SLICED=1: the split-8 level-5 ranges in one CTA per tile, BN 64, 72 chunks", 1, 22,
            40, 512, 128, 3, (64, 8), splits=1, ws="default", env={"SMOT_TC_SLICED": "1"}),
        _tc("sliced-2stage-lift", "SMOT_TC_SLICED=1 at the batch-10 2-stage shape: the 2-deep ring is lifted to 4", 10, 44,
            80, 256, 64, 3, (64, 4), splits=1, ws="default", env={"SMOT_TC_SLICED": "1"}),
    ]
    return c


def _refused_cases():
    """Descriptors the wgmma route refuses: SIMT (fp16) runs them."""
    return [
        Case("route-m15", "simt", "batch*OH*OW = 15 < 16: wgmma refuses; Cout 64 -> 64x64 tiles", 1, 3, 5, 64, 64, 3,
             ["conv_simt_kernel<half,half,64,64,4,4,1>"]),
        Case("route-cin96", "simt", "Cin 96 is not a multiple of 64: wgmma refuses (Cin % 16 == 0: vector form)", 1, 16, 32,
             96, 64, 1, ["conv_simt_kernel<half,half,64,64,4,4,1>"]),
        Case("route-in-ld-4mod64", "simt", "in_ld = 68 (4 mod 64): wgmma refuses (in_ld % 8); in_ld % 4 == 0: vector form",
             1, 16, 32, 64, 64, 3, ["conv_simt_kernel<half,half,64,64,4,4,1>"], in_ld=68, in_off=0),
        Case("route-out-ld-4mod64", "simt", "out_ld = 68: wgmma refuses (out_ld % 8)", 1, 16, 32, 64, 64, 3,
             ["conv_simt_kernel<half,half,64,64,4,4,1>"], out_ld=68, out_off=4),
        Case("route-in-8B", "simt", "input pointer 8-byte aligned (channel offset 4): wgmma refuses; SIMT scalar form", 1,
             16, 32, 64, 64, 3, ["conv_simt_kernel<half,half,64,64,4,4,0>"], in_ld=72, in_off=4),
        Case("route-s2-odd-h", "simt", "stride 2 with H = 21 odd: wgmma refuses", 1, 21, 40, 64, 64, 3,
             ["conv_simt_kernel<half,half,64,64,4,4,1>"], stride=2),
    ]


def _hires_cases():
    c = [Case("stem-odd-w", "hires", "stem 7x7 with W = 47 odd: the persistent stem needs even W, the per-tile kernel runs",
              1, 33, 47, 3, 16, 7, ["stem7x7_hires_kernel"], in_ld=4, in_off=0, in_fill="zero")]
    # every layer in both forms, ragged against its tile, batch 2, output into a channel slice with a wider pitch
    layers = (("stem", 3, 16, 7, 1, ("stem7x7_hires_kernel", "stem7x7_persist_kernel")),
              ("c16", 16, 16, 3, 1, ("conv3x3_hires_kernel<16,16,1>", "conv3x3_c16_persist_kernel")),
              ("s2-16-32", 16, 32, 3, 2, ("conv3x3_hires_kernel<16,32,2>", "conv3x3_s2_persist_kernel<16,32>")),
              ("s2-32-64", 32, 64, 3, 2, ("conv3x3_hires_kernel<32,64,2>", "conv3x3_s2_persist_kernel<32,64>")))
    for name, cin, cout, k, s, (tile, persist) in layers:
        # OH 37 / OW 45: ragged against 8 / 4 x 32 per-tile and 32 x 32 persistent tiles
        H, W = (37, 46) if s == 1 else (74, 90)
        kw = dict(in_ld=4, in_off=0, in_fill="zero") if name == "stem" else dict(in_ld=cin + 16, in_off=8)
        for mode, kern, form in (("0", tile, "per-tile"), ("2", persist, "persistent")):
            c.append(Case("hires-%s-%s" % (name, form), "hires",
                          "%s, %s form (SMOT_HIRES_PERSIST=%s), batch 2, OH/OW ragged, output slice at offset 16 of pitch %d"
                          % (name, form, mode, cout + 32), 2, H, W, cin, cout, k, [kern], stride=s, out_ld=cout + 32,
                          out_off=16, env={"SMOT_HIRES_PERSIST": mode}, **kw))
    # the persistent kernels' own loop: ntiles >= sm_count takes them by default, and with 150 or 180 tiles on at most 144
    # CTAs some CTAs run a second tile, in another image, prefetched into the other buffer; the map's last row and column of
    # tiles are ragged (OH 150 = 4 x 32 + 22, OW 166 = 5 x 32 + 6; OH 38 = 4 x 8 + 6 = 9 x 4 + 2, OW 165 = 5 x 32 + 5)
    for name, cin, cout, k, s, B, H, W, kern in (
            ("stem", 3, 16, 7, 1, 5, 150, 166, "stem7x7_persist_kernel"),
            ("c16", 16, 16, 3, 1, 5, 150, 166, "conv3x3_c16_persist_kernel"),
            ("s2-16-32", 16, 32, 3, 2, 5, 76, 330, "conv3x3_s2_persist_kernel<16,32>"),
            ("s2-32-64", 32, 64, 3, 2, 3, 76, 330, "conv3x3_s2_persist_kernel<32,64>")):
        kw = dict(in_ld=4, in_off=0, in_fill="zero") if name == "stem" else dict(in_ld=cin + 16, in_off=8)
        c.append(Case("hires-%s-persistent-loop" % name, "hires",
                      "%s, default route: %d tiles >= sm_count take the persistent form, more tiles than CTAs" % (name, (150 if
                      name != "s2-32-64" else 180)), B, H, W, cin, cout, k, [kern], stride=s, out_ld=cout + 32, out_off=16,
                      **kw))
    return c


def _sn(name, why, B, H, W, Cin, Cout, k, kern, dt="f16", odt=None, wk=None, **kw):
    return Case(name, "smalln", why, B, H, W, Cin, Cout, k, [kern], dt=dt, odt=odt, wk=wk, relu=False, **kw)


def _smalln_cases():
    return [
        # ---- mma.sync kernel (fp16 input, Cin % 32 == 0): NT = 1 for Cout <= 8, else 2; WK from the per-image K chunks
        _sn("sn-mma-c1-wk1", "mma, Cout 1 (NT 1); 1x1 Cin 64 = 2 chunks: WK 1", 1, 24, 40, 64, 1, 1,
            "conv_smalln_mma_kernel<half,1>", wk=1),
        _sn("sn-mma-c4-wk2", "mma, Cout 4; Cin 128 = 4 chunks: WK 2", 1, 24, 40, 128, 4, 1, "conv_smalln_mma_kernel<half,1>",
            wk=2),
        _sn("sn-mma-c5-wk4", "mma, Cout 5; Cin 256 = 8 chunks: WK 4", 1, 24, 40, 256, 5, 1, "conv_smalln_mma_kernel<half,1>",
            wk=4),
        _sn("sn-mma-c8-wk8", "mma, Cout 8; 3x3 Cin 64 = 18 chunks: WK 8", 1, 24, 40, 64, 8, 3, "conv_smalln_mma_kernel<half,1>",
            wk=8),
        _sn("sn-mma-c9-wk8", "mma, Cout 9 (NT 2), 3x3 Cin 64: WK 8", 2, 23, 41, 64, 9, 3, "conv_smalln_mma_kernel<half,2>",
            wk=8),
        _sn("sn-mma-c16-f32out", "mma, Cout 16, fp32 output into a pitched slice (offset 3, pitch 21)", 1, 24, 40, 128, 16, 3,
            "conv_smalln_mma_kernel<float,2>", odt="f32", wk=8, out_ld=21, out_off=3),
        # ---- direct kernel (M / batch <= 1024) and shared-memory kernel: fp32, or fp16 with Cin % 32 != 0
        _sn("sn-direct-c1", "direct, Cout 1 -> cout_pad 4; M = 1024", 1, 32, 32, 64, 1, 3,
            "conv_smalln_direct_kernel<float,float,4>", dt="f32"),
        _sn("sn-direct-c4", "direct, Cout 4 -> cout_pad 4", 1, 32, 32, 64, 4, 1, "conv_smalln_direct_kernel<float,float,4>",
            dt="f32"),
        _sn("sn-direct-c5", "direct, Cout 5 -> cout_pad 8", 1, 32, 32, 64, 5, 1, "conv_smalln_direct_kernel<float,float,8>",
            dt="f32"),
        _sn("sn-direct-c8", "direct, Cout 8 -> cout_pad 8", 1, 32, 32, 64, 8, 1, "conv_smalln_direct_kernel<float,float,8>",
            dt="f32"),
        _sn("sn-direct-c9", "direct, Cout 9 -> cout_pad 16", 1, 32, 32, 64, 9, 3, "conv_smalln_direct_kernel<float,float,16>",
            dt="f32"),
        _sn("sn-direct-batch2", "direct: 2 images of 1024 pixels (the threshold is per image)", 2, 32, 32, 64, 16, 3,
            "conv_smalln_direct_kernel<float,float,16>", dt="f32"),
        _sn("sn-smem-1025", "M / batch = 1025 > 1024: shared-memory kernel", 1, 25, 41, 64, 9, 3,
            "conv_smalln_kernel<float,float,16>", dt="f32"),
        _sn("sn-smem-c7", "M / batch = 1200 > 1024: shared-memory kernel, Cout 7 -> cout_pad 8", 1, 30, 40, 64, 7, 3,
            "conv_smalln_kernel<float,float,8>", dt="f32"),
        _sn("sn-smem-k1536", "K = 1536: 16 x K fp32 weights = 96 KB, the limit, accepted", 1, 40, 40, 1536, 4, 1,
            "conv_smalln_kernel<float,float,4>", dt="f32"),
        _sn("sn-f16-direct", "fp16 in / out, Cin 68 (not % 32: no mma), direct", 1, 20, 30, 68, 5, 3,
            "conv_smalln_direct_kernel<half,half,8>"),
        _sn("sn-f16-f32-smem", "fp16 in, fp32 out, Cin 68, M 1200: shared-memory kernel, fp32 pitched slice", 1, 30, 40, 68,
            16, 1, "conv_smalln_kernel<half,float,16>", odt="f32", out_ld=21, out_off=3),
        Case("sn-k1552-simt", "simt", "K = 1552 > the 96 KB limit: SIMT, Cout <= 16 tiles", 1, 40, 40, 1552, 4, 1,
             ["conv_simt_kernel<float,float,256,16,4,4,1>"], dt="f32", relu=False),
    ]


def _simt_cases():
    c = []
    for dt, odt in (("f32", "f32"), ("f16", "f16"), ("f16", "f32")):
        tag = "%s-%s" % (dt, odt)
        ti, to = ("float" if dt == "f32" else "half"), ("float" if odt == "f32" else "half")

        def k(cfg, vec):
            return "conv_simt_kernel<%s,%s,%s,%d>" % (ti, to, cfg, vec)
        c += [
            Case("simt-m8191-" + tag, "simt", "M = 8191 < 8192: 64x64 tiles", 1, 1, 8191, 48, 64, 1, [k("64,64,4,4", 1)],
                 dt=dt, odt=odt),
            Case("simt-m8192-" + tag, "simt", "M = 8192: 128x64 tiles", 1, 64, 128, 48, 64, 1, [k("128,64,8,4", 1)], dt=dt,
                 odt=odt),
            Case("simt-s2-cout16-" + tag, "simt", "Cout 16 with stride 2 (small-N refuses stride 2)", 1, 30, 41, 64, 16, 3,
                 [k("256,16,4,4", 1)], stride=2, dt=dt, odt=odt),
            Case("simt-res-cout5-" + tag, "simt", "Cout 5 with a residual (small-N refuses residuals)", 2, 17, 23, 64, 5, 3,
                 [k("256,16,4,4", 1)], res=True, dt=dt, odt=odt),
            Case("simt-vec-" + tag, "simt", "vector form: Cin 48 % 16 == 0, in_ld % 4 == 0, 16-byte pointers", 1, 19, 37, 48,
                 72, 3, [k("64,64,4,4", 1)], res=True, dt=dt, odt=odt),
            Case("simt-scalar-cin-" + tag, "simt", "scalar form: Cin 40 is not a multiple of the K tile (16)", 1, 19, 37, 40,
                 72, 3, [k("64,64,4,4", 0)], res=True, dt=dt, odt=odt),
            Case("simt-scalar-ld-" + tag, "simt", "scalar form: in_ld 53 odd", 1, 19, 37, 48, 72, 3, [k("64,64,4,4", 0)],
                 in_ld=53, in_off=5, dt=dt, odt=odt),
            Case("simt-scalar-ptr-" + tag, "simt", "scalar form: input pointer 4 bytes past 16-byte alignment", 1, 19, 37, 48,
                 72, 3, [k("64,64,4,4", 0)], in_ld=56, in_off=(1 if dt == "f32" else 2), dt=dt, odt=odt),
            Case("simt-scalar-m8192-" + tag, "simt", "scalar form of the 128x64 tiles: Cin 3", 1, 64, 128, 3, 64, 3,
                 [k("128,64,8,4", 0)], in_ld=3, in_off=0, dt=dt, odt=odt),
            Case("simt-scalar-cout16-" + tag, "simt", "scalar form of the Cout <= 16 tiles: Cin 3, 7x7 pad 3", 1, 33, 47, 3,
                 16, 7, [k("256,16,4,4", 0)], in_ld=3, in_off=0, dt=dt, odt=odt, relu=False),
            Case("simt-1x1-s2-" + tag, "simt", "1x1 with stride 2 (OH 12, OW 19 from 23 x 37)", 1, 23, 37, 64, 64, 1,
                 [k("64,64,4,4", 1)], stride=2, dt=dt, odt=odt),
        ]
    return c


def all_cases():
    return _wgmma_cases() + _refused_cases() + _hires_cases() + _smalln_cases() + _simt_cases()


CASES = all_cases()
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES), "duplicate case names"


def child_cases():
    """Cases that need a switch read once per process (SMOT_TC_CLUSTER, SMOT_TC_MAXSPLIT): run in a child process."""
    return {
        # the cluster finish, against the reduce path bit for bit; both routes to a 2-stage ring
        "cluster": dict(env={"SMOT_TC_CLUSTER": "1"}, cases=[
            ("split-8-level5", None), ("split-3", None), ("fc6-300", None), ("split-empty-rounding", None),
            ("s2-split", None), ("split-batch10-2stage", None), ("split-8-level5", {"SMOT_TC_STAGES": "2"})]),
        # the split factor the default rule never produces
        "maxsplit2": dict(env={"SMOT_TC_MAXSPLIT": "2"}, cases=[("split-8-level5", None), ("fc6-30", None)]),
    }


# ------------------------------------------------------------------------------------------------------------------------
# operands in guarded buffers
# ------------------------------------------------------------------------------------------------------------------------
def _int_view(t):
    return t.view(torch.int16 if t.dtype == F16 else torch.int32)


def _guarded(n_pix, ld, off, width, dtype, device, fill="nan"):
    """A flat buffer of MARGIN + n_pix * ld + MARGIN elements, NaN-pattern (or zero) filled; returns (buffer, view of the
    (n_pix, width) operand at channel offset `off` with pixel pitch `ld`)."""
    buf = torch.empty(MARGIN + n_pix * ld + MARGIN, dtype=dtype, device=device)
    if fill == "nan":
        _int_view(buf).fill_(NAN_BITS[dtype])
    else:
        buf.zero_()
    view = buf[MARGIN + off:].as_strided((n_pix, width), (ld, 1))
    return buf, view


def _chunk_edges(n):
    """The first and last channel of every 64-channel chunk, and the last channel."""
    e = set()
    for c0 in range(0, n, 64):
        e.add(c0)
        e.add(min(c0 + 63, n - 1))
    e.add(n - 1)
    return sorted(e)


def make_operands(case, pattern, device, seed=None):
    """Host-generated fp64 operand values (rounded to their storage dtype) of one case; returns a dict."""
    g = torch.Generator().manual_seed(seed if seed is not None else (zlib.crc32(case.name.encode()) & 0xFFFF) * 2 + (pattern == "exact"))
    B, H, W, Cin, Cout, k = case.B, case.H, case.W, case.Cin, case.Cout, case.k
    OH, OW = case.OH, case.OW
    if pattern == "gauss":
        x = torch.randn(B, H, W, Cin, generator=g, dtype=torch.float64)
        w = torch.randn(Cout, k, k, Cin, generator=g, dtype=torch.float64) / (case.K ** 0.5)
        scale = 0.5 + torch.rand(Cout, generator=g, dtype=torch.float64)
        bias = 0.5 * torch.randn(Cout, generator=g, dtype=torch.float64)
        res = torch.randn(B, OH, OW, Cout, generator=g, dtype=torch.float64) if case.res else None
    else:
        def sparse(shape, p, vals):
            v = torch.tensor(vals, dtype=torch.float64)[torch.randint(len(vals), shape, generator=g)]
            return v * (torch.rand(shape, generator=g) < p)
        x = sparse((B, H, W, Cin), 0.12, [-2, -1, 1, 2])
        e = torch.tensor(_chunk_edges(Cin))
        sgn = lambda shape: torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double()  # noqa: E731
        x[:, H - 1, :, e] = sgn((B, W, len(e)))            # last row of each image
        x[:, :, W - 1, e] = sgn((B, H, len(e)))            # last column
        w = sparse((Cout, k, k, Cin), 0.12, [-1, 1])
        w[:, :, :, e] = sgn((Cout, k, k, len(e))) * (torch.rand(Cout, k, k, len(e), generator=g) < 0.5)
        w[:, k - 1, k - 1, e] = sgn((Cout, len(e)))        # the last tap, every chunk edge
        scale = torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64)[torch.randint(3, (Cout,), generator=g)]
        bias = torch.randint(-8, 9, (Cout,), generator=g).double()
        res = sparse((B, OH, OW, Cout), 0.5, [-3, -1, 1, 2]) if case.res else None
    x, w = x.to(case.dt), w.to(case.dt)
    scale, bias = scale.float(), bias.float()
    res = res.to(case.dt) if res is not None else None
    if pattern == "exact":
        xc, wc = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
        mag = F.conv2d(xc.abs(), wc.abs(), None, case.stride, case.pad)
        tot = mag * scale.double().view(1, -1, 1, 1) + bias.double().abs().view(1, -1, 1, 1)
        if res is not None:
            tot = tot + res.double().abs().permute(0, 3, 1, 2)
        assert float(mag.max()) < 2 ** 11 and float(tot.max()) < 2 ** 10, "%s: exact operands too large" % case.name
    return dict(x=x, w=w, scale=scale, bias=bias, res=res)


class Placed(object):
    """One case's operands in guarded buffers on `device`, and its descriptor."""

    def __init__(self, case, ops, device):
        from siammot_b200 import _lib
        self.case = case
        dev = torch.device(device)
        B, OH, OW = case.B, case.OH, case.OW
        npix_in, npix_out = B * case.H * case.W, B * OH * OW
        self.in_buf, xin = _guarded(npix_in, case.in_ld, case.in_off, case.Cin, case.dt, dev, case.in_fill)
        xin.copy_(ops["x"].reshape(npix_in, case.Cin))
        self.w = ops["w"].contiguous().to(dev)
        self.scale, self.bias = ops["scale"].to(dev), ops["bias"].to(dev)
        self.out_buf, self.out_view = _guarded(npix_out, case.out_ld, case.out_off, case.Cout, case.odt, dev)
        self.res_buf = None
        if case.res:
            self.res_buf, rv = _guarded(npix_out, case.res_ld, case.res_off, case.Cout, case.dt, dev)
            rv.copy_(ops["res"].reshape(npix_out, case.Cout))
        self.ws = None
        if case.ws:
            self.ws = torch.zeros(case.ws, dtype=torch.uint8, device=dev)
            self.ws[:WS_COUNTER].fill_(WS_BYTE)
        ei, eo = self.in_buf.element_size(), self.out_buf.element_size()
        d = self.d = _lib.ConvDesc()
        d.inp = self.in_buf.data_ptr() + (MARGIN + case.in_off) * ei
        d.weight, d.scale, d.bias = self.w.data_ptr(), self.scale.data_ptr(), self.bias.data_ptr()
        d.residual = self.res_buf.data_ptr() + (MARGIN + case.res_off) * ei if case.res else None
        d.out = self.out_buf.data_ptr() + (MARGIN + case.out_off) * eo
        d.batch, d.H, d.W, d.Cin, d.in_ld = B, case.H, case.W, case.Cin, case.in_ld
        d.OH, d.OW, d.Cout, d.out_ld, d.res_ld = OH, OW, case.Cout, case.out_ld, case.res_ld
        d.KH = d.KW = case.k
        d.stride, d.pad, d.relu = case.stride, case.pad, int(case.relu)
        d.in_dtype, d.out_dtype, d.algo = CODE[case.dt], CODE[case.odt], 0
        d.workspace = self.ws.data_ptr() if self.ws is not None else None
        d.workspace_bytes = case.ws or 0
        self.before = dict(inp=self.in_buf.clone(), out=self.out_buf.clone(),
                           res=self.res_buf.clone() if self.res_buf is not None else None)

    def output(self):
        return self.out_view.reshape(self.case.B, self.case.OH, self.case.OW, self.case.Cout)

    def guard_faults(self):
        """Names of the guarded regions that changed."""
        bad = []
        if not torch.equal(_int_view(self.in_buf), _int_view(self.before["inp"])):
            bad.append("input")
        if self.res_buf is not None and not torch.equal(_int_view(self.res_buf), _int_view(self.before["res"])):
            bad.append("residual")
        post, pre = _int_view(self.out_buf.clone()), _int_view(self.before["out"].clone())
        c = self.case
        for t in (post, pre):
            t[MARGIN + c.out_off:].as_strided((c.B * c.OH * c.OW, c.Cout), (c.out_ld, 1)).zero_()
        if not torch.equal(post, pre):
            idx = int((post != pre).nonzero()[0]) - MARGIN
            bad.append("output outside the operand (element %d from the operand base: pixel %d, channel %d)"
                       % (idx - c.out_off, (idx - c.out_off) // c.out_ld, (idx - c.out_off) % c.out_ld))
        if self.ws is not None and not bool((self.ws[:WS_COUNTER] == WS_BYTE).all()):
            bad.append("workspace counter bytes")
        return bad


class Result(object):
    def __init__(self, case, pattern):
        self.case, self.pattern = case, pattern
        self.max_ratio, self.max_err, self.where, self.exact_ok, self.guards = 0.0, 0.0, None, None, []
        self.kernels, self.output = None, None

    @property
    def ok(self):
        return self.max_ratio <= 1.0 and self.exact_ok is not False and not self.guards

    def describe(self):
        return ("%s/%s: |err|/bound %.3f%s%s%s" % (self.case.name, self.pattern, self.max_ratio,
                "" if self.exact_ok is None else (", bit-exact" if self.exact_ok else ", NOT bit-exact"),
                (" guards changed: %s" % self.guards) if self.guards else "",
                (" worst at %s" % (self.where,)) if not self.ok else ""))


def run_case(case, pattern, device, launch, ops=None, keep_output=False):
    """Place, snapshot, launch(placed), compare.  launch(p) runs the convolution of p.d (on the GPU: smot_conv2d)."""
    ops = ops if ops is not None else make_operands(case, pattern, device)
    p = Placed(case, ops, device)
    mem = lc.Memory(device)
    snap = lc.conv_snapshot(mem, p.d)
    launch(p)
    y = mem.nhwc(p.d.out, case.B, case.OH, case.OW, case.Cout, case.out_ld, case.odt)
    r, b = lc.conv_reference(*snap[:2], p.d, *snap[2:])
    res = Result(case, pattern)
    ck = lc.Check()
    ck.bound("out", y, r, b)
    res.max_ratio, res.max_err, res.where = ck.max_ratio, ck.max_err, ck.where
    if pattern == "exact":
        ex = lc.Check()
        ex.exact("out", y, r)
        res.exact_ok = ex.max_ratio == 0.0
        if not res.exact_ok:
            res.where = ex.where
    res.guards = p.guard_faults()
    if keep_output:
        res.output = p.output().detach().cpu().clone()
    return res


# ------------------------------------------------------------------------------------------------------------------------
# kernel names seen by torch.profiler
# ------------------------------------------------------------------------------------------------------------------------
def kernel_id(name):
    """'void smot::conv_tc_kernel<(int)128, (int)2>(CUtensorMap_st, ...)' -> 'conv_tc_kernel<128,2>'; None for kernels
    outside the smot namespace."""
    if "smot::" not in name:
        return None
    s = name[5:] if name.startswith("void ") else name
    depth = 0
    for i, ch in enumerate(s):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            s = s[:i]
            break
    s = s.replace("smot::", "")
    s = re.sub(r"\((?:int|bool|unsigned int|unsigned)\)", "", s)
    s = re.sub(r"\s+", "", s).replace("__half", "half").replace("true", "1").replace("false", "0")
    return s


def profiled(fn):
    """Run fn() under torch.profiler (CPU and CUDA activities); returns [(kernel id, grid)] of the smot kernels in launch order.
    The profiler now and then delivers no kernel record at all: fn() (a convolution that rewrites its output from the same
    operands) is then run again, up to five times in all."""
    for _ in range(5):
        out = _profiled_once(fn)
        if out:
            break
    return out


def _profiled_once(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            tr = json.load(f)
    ev = [e for e in tr.get("traceEvents", []) if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e.get("ts", 0))
    out = []
    for e in ev:
        kid = kernel_id(e.get("name", ""))
        if kid is not None:
            out.append((kid, tuple(e.get("args", {}).get("grid", ()))))
    return out


def expected_grid_check(case, launched):
    """Problems with the split factor (conv_tc_kernel grid.z) or the small-N K slicing (mma grid.x) of a launch list."""
    errs = []
    for kid, grid in launched:
        if case.splits is not None and kid.startswith("conv_tc_kernel") and grid and grid[2] != case.splits:
            errs.append("%s grid %s: expected %d K splits" % (kid, grid, case.splits))
        if case.wk is not None and kid.startswith("conv_smalln_mma_kernel") and grid:
            mtiles = -(-case.B * case.OH * case.OW // 16)
            want = -(-mtiles // (8 // case.wk))
            if grid[0] != want:
                errs.append("%s grid %s: expected WK %d (grid.x %d)" % (kid, grid, case.wk, want))
    return errs


def gpu_launch(p):
    from siammot_b200 import _lib
    rc = _lib.lib().smot_conv2d(C.byref(p.d), _lib.stream_ptr())
    torch.cuda.synchronize()
    _lib.check(rc, "smot_conv2d(%s)" % p.case.name)


def gpu_algo(p):
    from siammot_b200 import _lib
    return int(_lib.lib().smot_conv2d_algo(C.byref(p.d)))
