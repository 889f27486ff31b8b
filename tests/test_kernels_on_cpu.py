"""Source text of the simple kernels written without GPU access, executed on the host (tests/cpu_cuda/shim.h: a block's threads
are OS threads, __syncthreads is a barrier) and compared with the oracle / the C-ABI emulator's specification:
roi_align_planar_kernel<float>, maxpool3x3s2_kernel<float>, track_combine_grouped_kernel.  The tensor-core / bulk-copy kernel
(xcorr_planar_kernel) cannot be run this way and stays GPU-only."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "cpu_cuda"))


@pytest.fixture(scope="module")
def cpu_kernels():
    import cpu_cuda_build as cpu_build
    return C.CDLL(cpu_build.build())


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


@pytest.mark.parametrize("res,row_pitch,plane", [(30, 40, 1208), (15, 16, 240)])
def test_roi_align_planar_kernel_source_matches_oracle(cpu_kernels, res, row_pitch, plane):
    from oracle import siammot_oracle as orc
    from siammot_b200._lib import Pyramid
    g = torch.Generator().manual_seed(3)
    Cc, H, W = 136, 24, 40                 # two channel passes per lane (c += 128) and a ragged last one
    feats = [torch.randn(1, Cc, H >> i, W >> i, generator=g) for i in range(4)]
    nhwc = [f.permute(0, 2, 3, 1).contiguous() for f in feats]
    boxes = torch.tensor([[10., 20., 60., 90.], [-30., -20., 40., 50.], [5., 5., 150., 90.], [100., 30., 158., 95.], [70., 10., 71., 11.]])
    pad = 64
    sr = orc.search_region(boxes, pad, 1.0, 0)
    pads = [int(pad / ((2 ** i) * 4)) for i in range(4)]
    pyr = Pyramid()
    pyr.num_levels, pyr.k_min = 4, 2
    for l in range(4):
        pyr.feat[l], pyr.H[l], pyr.W[l], pyr.ld[l] = nhwc[l].data_ptr(), H >> l, W >> l, Cc
        pyr.scale[l], pyr.pad[l] = 0.25 / (2 ** l), pads[l]
    n = boxes.shape[0]
    count = torch.tensor([4], dtype=torch.int32)      # the last roi is past the device-side count: zero rows
    out = torch.full((n, Cc, plane), 7.0)
    cpu_kernels.cpu_roi_align_planar(C.byref(pyr), p(sr), p(boxes), p(count), n, Cc, res, 2, p(out), row_pitch, plane)
    ref = orc.pool_rois(orc.pad_features(feats, pad), boxes[:4], boxes[:4], (0.25, 0.125, 0.0625, 0.03125), res, 2, rois=sr[:4])
    # the GPU-validated NHWC kernel through the same shim: same arithmetic, so the two kernels must agree exactly (this also
    # validates the shim on a kernel whose GPU behaviour is known)
    nhwc_out = torch.full((n, res, res, Cc), 7.0)
    cpu_kernels.cpu_roi_align(C.byref(pyr), p(sr), p(boxes), p(count), n, Cc, res, 2, p(nhwc_out))
    assert float((nhwc_out[:4].permute(0, 3, 1, 2) - ref).abs().max()) <= 2e-5 * float(ref.abs().max())
    assert torch.equal(out[:, :, :res * row_pitch].reshape(n, Cc, res, row_pitch)[..., :res], nhwc_out.permute(0, 3, 1, 2))
    rows = out[:, :, :res * row_pitch].reshape(n, Cc, res, row_pitch)
    got = rows[..., :res]
    assert float((got[:4] - ref).abs().max()) <= 2e-5 * float(ref.abs().max())
    assert float(got[4].abs().max()) == 0.0                                   # past the count
    assert float((rows[..., res:] - 7.0).abs().max()) == 0.0                  # pad columns never written
    assert float((out[:, :, res * row_pitch:] - 7.0).abs().max()) == 0.0 if plane > res * row_pitch else True
    # the row-wise kernel with separable sample tables (round 2, the default): bit-identical to both, NHWC and planar
    rows_nhwc = torch.full((n, res, res, Cc), 7.0)
    cpu_kernels.cpu_roi_align_rows(C.byref(pyr), p(sr), p(boxes), p(count), n, Cc, res, 2, p(rows_nhwc), 0, 0, 0)
    assert torch.equal(rows_nhwc, nhwc_out)
    rows_planar = torch.full((n, Cc, plane), 7.0)
    cpu_kernels.cpu_roi_align_rows(C.byref(pyr), p(sr), p(boxes), p(count), n, Cc, res, 2, p(rows_planar), row_pitch, plane, 1)
    assert torch.equal(rows_planar, out)
    # ... and without the padded frame (the box head's / template pooler's use: pads 0, rois = level boxes)
    for l in range(4):
        pyr.pad[l] = 0
    a1, a2 = torch.full((n, res, res, Cc), 7.0), torch.full((n, res, res, Cc), 7.0)
    cpu_kernels.cpu_roi_align(C.byref(pyr), p(boxes), None, None, n, Cc, res, 2, p(a1))
    cpu_kernels.cpu_roi_align_rows(C.byref(pyr), p(boxes), None, None, n, Cc, res, 2, p(a2), 0, 0, 0)
    assert torch.equal(a1, a2)
    a3 = torch.full((n, res, res, Cc), 7.0)
    cpu_kernels.cpu_roi_align_rows(C.byref(pyr), p(boxes), None, None, n, Cc, res, 2, p(a3), 0, 0, 2)   # unrolled specialisation
    assert torch.equal(a1, a3)
    for small in (7, 3):                                  # several bin rows per CTA (the box head's 7 x 7: the whole roi)
        b1, b2 = torch.full((n, small, small, Cc), 7.0), torch.full((n, small, small, Cc), 7.0)
        cpu_kernels.cpu_roi_align(C.byref(pyr), p(boxes), None, p(count), n, Cc, small, 2, p(b1))
        cpu_kernels.cpu_roi_align_rows(C.byref(pyr), p(boxes), None, p(count), n, Cc, small, 2, p(b2), 0, 0, 0)
        assert torch.equal(b1, b2)


def test_maxpool3x3s2_kernel_source_matches_torch(cpu_kernels):
    g = torch.Generator().manual_seed(4)
    for B, Cc, H, W in ((1, 8, 13, 18), (2, 4, 6, 5), (1, 12, 1, 7)):
        x = torch.randn(B, Cc, H, W, generator=g)
        ref = F.max_pool2d(x, 3, 2, 1)
        xin = torch.zeros(B, H, W, Cc + 4)
        xin[..., 4:] = x.permute(0, 2, 3, 1)
        out = torch.full((B, ref.shape[2], ref.shape[3], Cc + 8), 7.0)
        cpu_kernels.cpu_maxpool3x3s2(C.c_void_p(xin.data_ptr() + 16), C.c_void_p(out.data_ptr() + 16), B, H, W, Cc, Cc + 4, Cc + 8)
        assert torch.equal(out[..., 4:4 + Cc].permute(0, 3, 1, 2), ref)
        assert float((out[..., :4] - 7.0).abs().max()) == 0.0 and float((out[..., 4 + Cc:] - 7.0).abs().max()) == 0.0


def test_track_combine_grouped_kernel_source_matches_specification(cpu_kernels):
    import cabi_emulator as ce
    spec = ce.FakeLib()
    rng = np.random.default_rng(1)
    for trial in range(60):
        n, ncap, ncls = int(rng.integers(1, 70)), int(rng.integers(0, 40)), int(rng.integers(3, 6))
        tracktor = int(rng.integers(0, 2))
        src = dict(det_boxes=torch.rand(max(ncap, 1), 4), det_scores=torch.rand(max(ncap, 1)), dec_boxes=torch.rand(n, ncls, 4),
                   dec_scores=torch.rand(n, ncls), labels=torch.tensor(rng.integers(1, ncls, n), dtype=torch.int32),
                   conf=torch.rand(n), valid=torch.tensor(rng.integers(0, 2, n), dtype=torch.int32),
                   active=torch.tensor(rng.integers(0, 2, n), dtype=torch.float32))
        outs = []
        for which in ("spec", "kernel"):
            o = dict(cb=torch.full((ncap + n, 4), 9.), cs=torch.full((ncap + n,), 9.), zc=torch.tensor([5], dtype=torch.int32),
                     perm=torch.full((n,), 7, dtype=torch.int32))
            args = (p(src["det_boxes"]), p(src["det_scores"]), ncap, p(src["dec_boxes"]), p(src["dec_scores"]), ncls, p(src["labels"]),
                    p(src["conf"]), p(src["valid"]), p(src["active"]), n, tracktor, p(o["cb"]), p(o["cs"]), p(o["zc"]), p(o["perm"]))
            if which == "spec":
                spec.smot_track_combine_grouped(*args, None)
            else:
                cpu_kernels.cpu_track_combine_grouped(*args)
            outs.append(o)
        for k in outs[0]:
            assert torch.equal(outs[0][k], outs[1][k]), (trial, k)


@pytest.fixture(scope="module")
def cpu_xcorr():
    import cpu_cuda_build as cpu_build
    if not os.path.exists(os.path.join(cpu_build.CUDA_INCLUDE, "cuda_fp16.h")):
        pytest.skip("CUDA headers not found (cuda_fp16.h is compiled in host mode)")
    return C.CDLL(cpu_build.build_xcorr())


@pytest.mark.parametrize("n,Cc", [(2, 32), (1, 16), (3, 48)])
def test_xcorr_kernels_source_under_ptx_emulation(cpu_xcorr, n, Cc):
    """csrc/emm.cu's tensor-core correlation kernels, source text, with ldmatrix / mma.sync / mbarrier / cp.async.bulk emulated
    on the host (tests/cpu_cuda/shim_tc.h).  xcorr_mma_kernel is validated on the GPU: its agreement with the oracle here
    validates the emulation.  xcorr_planar_kernel (written without GPU access: bulk-copy staging from channel-planar windows,
    17th warp, mbarrier) must then reproduce xcorr_mma_kernel's output bit for bit."""
    from oracle import siammot_oracle as orc
    from siammot_b200 import _lib
    g = torch.Generator().manual_seed(n * 100 + Cc)
    x = torch.randn(n, Cc, 30, 30, generator=g).half()
    k = (torch.randn(n, Cc, 15, 15, generator=g) / 15.).half()
    ref = orc.xcorr_depthwise(x.float(), k.float())
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    k_nhwc = k.permute(0, 2, 3, 1).contiguous()
    out_mma = torch.zeros(n, 16, 16, Cc, dtype=torch.float16)
    cpu_xcorr.cpu_xcorr_mma(p(x_nhwc), p(k_nhwc), p(out_mma), n, Cc)
    err = float((out_mma.permute(0, 3, 1, 2).float() - ref).abs().max() / ref.abs().max())
    assert err <= 2e-3, "emulated xcorr_mma_kernel vs oracle: %g" % err
    PL, RP = _lib.XCORR_PLANE, _lib.XCORR_ROW_PITCH
    assert cpu_xcorr.cpu_xcorr_plane_halves() == PL
    xp = torch.full((n, Cc, PL), 77.0, dtype=torch.float16)                    # never-read halves hold garbage
    rows = xp[:, :, :30 * RP].view(n, Cc, 30, RP)
    rows[..., :30] = x
    rows[..., 30:32] = 0.0                                                     # the producer's zero columns
    out_planar = torch.zeros(n, 16, 16, Cc, dtype=torch.float16)
    cpu_xcorr.cpu_xcorr_planar(p(xp), p(k_nhwc), p(out_planar), n, Cc, 0)
    assert torch.equal(out_planar, out_mma)
    # MMA_MODE 1 (SMOT_XCORR_PLANAR=2): m16n8k8 on the live halves, fragments shared between template rows u and u+8 --
    # another accumulation order, so equality holds to fp16 rounding: the oracle bar, and at most one fp16 ulp from mode 0
    out_trim = torch.zeros(n, 16, 16, Cc, dtype=torch.float16)
    cpu_xcorr.cpu_xcorr_planar(p(xp), p(k_nhwc), p(out_trim), n, Cc, 1)
    err = float((out_trim.permute(0, 3, 1, 2).float() - ref).abs().max() / ref.abs().max())
    assert err <= 2e-3, "emulated trimmed planar kernel vs oracle: %g" % err
    d = (out_trim.float() - out_mma.float()).abs()
    assert float((d / out_mma.float().abs().clamp_min(2e-2)).max()) <= 1.1e-3      # one fp16 ulp (2^-10) of the larger values
    assert float((d > 0).float().mean()) < 0.05                                    # and rare
    # the channel group of a CTA (planes = MMA warps: 2 / 4 / 8 / 16) only sets the grid: the results are the same bits
    for cg in ((2, 4, 8) if n * Cc <= 64 else (8,)):      # (the big case keeps the suite's run time down: one group only)
        for mode, want in ((0, out_mma), (1, out_trim)):
            got = torch.full((n, 16, 16, Cc), float("nan"), dtype=torch.float16)
            assert cpu_xcorr.cpu_xcorr_planar_cfg(p(xp), p(k_nhwc), p(got), n, Cc, mode, cg) == 0
            assert torch.equal(got, want), "channel group %d, mode %d" % (cg, mode)
    # flat form (one CTA per SM, the plane list dealt in 4-plane units): CTAs of 4-5 units, some straddling a track boundary, a
    # single CTA, and one unit per CTA -- the same bits again
    for grid in sorted({(n * Cc // 4 + 4) // 5} | ({1, n * Cc // 4} if n * Cc <= 28 else set())):
        for mode, want in ((0, out_mma), (1, out_trim)):
            got = torch.full((n, 16, 16, Cc), float("nan"), dtype=torch.float16)
            assert cpu_xcorr.cpu_xcorr_flat(p(xp), p(k_nhwc), p(got), n, Cc, mode, grid) == 0
            assert torch.equal(got, want), "flat form, grid %d, mode %d" % (grid, mode)


def test_fp16_instantiations_of_the_simple_kernels(cpu_xcorr):
    """The fp16 instantiations the fp16 engine actually launches: planar ROIAlign == the validated NHWC kernel bit for bit,
    3x3/2 max-pool == torch."""
    from oracle import siammot_oracle as orc
    from siammot_b200 import _lib
    from siammot_b200._lib import Pyramid
    g = torch.Generator().manual_seed(9)
    Cc, H, W = 32, 24, 40
    feats = [torch.randn(1, Cc, H >> i, W >> i, generator=g).half() for i in range(4)]
    nhwc = [f.permute(0, 2, 3, 1).contiguous() for f in feats]
    boxes = torch.tensor([[10., 20., 60., 90.], [-30., -20., 40., 50.], [100., 30., 158., 95.]])
    pad = 64
    sr = orc.search_region(boxes, pad, 1.0, 0)
    pyr = Pyramid()
    pyr.num_levels, pyr.k_min = 4, 2
    for l in range(4):
        pyr.feat[l], pyr.H[l], pyr.W[l], pyr.ld[l] = nhwc[l].data_ptr(), H >> l, W >> l, Cc
        pyr.scale[l], pyr.pad[l] = 0.25 / (2 ** l), int(pad / ((2 ** l) * 4))
    n, res, RP, PL = 3, 30, _lib.XCORR_ROW_PITCH, _lib.XCORR_PLANE
    ref = torch.zeros(n, res, res, Cc, dtype=torch.float16)
    cpu_xcorr.cpu_roi_align_h(C.byref(pyr), p(sr), p(boxes), None, n, Cc, res, 2, p(ref))
    want = orc.pool_rois(orc.pad_features([f.float() for f in feats], pad), boxes, boxes, (0.25, 0.125, 0.0625, 0.03125), res, 2, rois=sr)
    assert float((ref.permute(0, 3, 1, 2).float() - want).abs().max()) <= 2e-3 * float(want.abs().max())
    planes = torch.zeros(n, Cc, PL, dtype=torch.float16)
    cpu_xcorr.cpu_roi_align_planar_h(C.byref(pyr), p(sr), p(boxes), None, n, Cc, res, 2, p(planes), RP, PL)
    rows = planes[:, :, :res * RP].view(n, Cc, res, RP)
    assert torch.equal(rows[..., :res], ref.permute(0, 3, 1, 2))
    assert float(rows[..., res:].abs().max()) == 0.0 and float(planes[:, :, res * RP:].abs().max()) == 0.0
    # the row-wise kernel (separable sample tables), fp16 instantiation: bit-identical to both
    r_nhwc = torch.zeros(n, res, res, Cc, dtype=torch.float16)
    cpu_xcorr.cpu_roi_align_rows_h(C.byref(pyr), p(sr), p(boxes), None, n, Cc, res, 2, p(r_nhwc), 0, 0, 0)
    assert torch.equal(r_nhwc, ref)
    r_planes = torch.zeros(n, Cc, PL, dtype=torch.float16)
    cpu_xcorr.cpu_roi_align_rows_h(C.byref(pyr), p(sr), p(boxes), None, n, Cc, res, 2, p(r_planes), RP, PL, 1)
    assert torch.equal(r_planes, planes)
    x = torch.randn(1, 8, 9, 14, generator=g).half()
    out = torch.zeros(1, 5, 7, 8, dtype=torch.float16)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()       # keep it alive across the call
    cpu_xcorr.cpu_maxpool3x3s2_h(p(x_nhwc), p(out), 1, 9, 14, 8, 8, 8)
    assert torch.equal(out.permute(0, 3, 1, 2), F.max_pool2d(x.float(), 3, 2, 1).half())


@pytest.mark.parametrize("stride", [1, 2])
def test_deform_im2col_kernel_source_matches_torchvision(cpu_kernels, cpu_xcorr, stride):
    """deform_im2col3x3_kernel (DCN v1 sampling) + a GEMM over its columns == torchvision.ops.deform_conv2d; fp32 and fp16
    instantiations; channel pitches wider than the channel counts."""
    from torchvision.ops import deform_conv2d
    g = torch.Generator().manual_seed(stride)
    Cc, H, W = 8, 11, 14
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    x = torch.randn(1, Cc, H, W, generator=g)
    w = torch.randn(6, Cc, 3, 3, generator=g)
    off = torch.randn(1, 18, OH, OW, generator=g) * 2.0
    ref = deform_conv2d(x, off, w, None, stride=stride, padding=1)
    off_nhwc = torch.zeros(1, OH, OW, 20)
    off_nhwc[..., :18] = off.permute(0, 2, 3, 1)
    for dtype, fn, tol_ in ((torch.float32, cpu_kernels.cpu_deform_im2col3x3, 1e-5), (torch.float16, cpu_xcorr.cpu_deform_im2col3x3_h, 4e-3)):
        xin = torch.zeros(1, H, W, Cc + 4, dtype=dtype)
        xin[..., :Cc] = x.permute(0, 2, 3, 1).to(dtype)
        cols = torch.full((1, OH, OW, 9 * Cc + 4), 7.0, dtype=dtype)
        fn(p(xin), p(off_nhwc), p(cols), H, W, Cc, Cc + 4, 20, OH, OW, 9 * Cc + 4, stride)
        assert float((cols[..., 9 * Cc:].float() - 7.0).abs().max()) == 0.0
        wq = w.permute(0, 2, 3, 1).reshape(6, 9 * Cc).to(dtype).float()            # [Cout][(tap, channel)], the engine's GEMM view
        got = torch.einsum("hwk,ok->ohw", cols[0, :, :, :9 * Cc].float(), wq)[None]
        want = ref if dtype == torch.float32 else deform_conv2d(x.half().float(), off, w.half().float(), None, stride=stride, padding=1)
        assert float((got - want).abs().max()) <= tol_ * float(want.abs().max())


@pytest.fixture(scope="module")
def cpu_hires():
    import cpu_cuda_build as cpu_build
    if not os.path.exists(os.path.join(cpu_build.CUDA_INCLUDE, "cuda_fp16.h")):
        pytest.skip("CUDA headers not found (cuda_fp16.h is compiled in host mode)")
    return C.CDLL(cpu_build.build_hires())


@pytest.mark.parametrize("H,W,batch,ctas", [(100, 130, 1, 6), (40, 70, 2, 3)])
def test_persistent_hires_kernels_reproduce_the_per_tile_kernels(cpu_hires, H, W, batch, ctas):
    """csrc/conv_hires.cu: stem 7x7 3->16 and level0 3x3 16->16.  The per-tile kernels are validated on the GPU (oracle bar);
    here they also meet torch's convolution, which validates the emulation, and the persistent forms (weights as register-resident
    B fragments, a warp owns four output rows, double-buffered halo, several tiles per CTA, ragged right / bottom tiles, two
    images) must equal them bit for bit -- garbage in the output pitch's unused channels stays untouched."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(H * W + batch)
    # ---- stem
    x = torch.randn(batch, 3, H, W, generator=g).half()
    w = (torch.randn(16, 3, 7, 7, generator=g) / 12.).half()
    scale, bias = torch.rand(16, generator=g) + 0.5, torch.randn(16, generator=g) * 0.1
    x_nhwc = torch.zeros(batch, H, W, 4, dtype=torch.float16)
    x_nhwc[..., :3] = x.permute(0, 2, 3, 1)
    w_k = w.permute(0, 2, 3, 1).contiguous()                                  # [Cout][KH][KW][Cin]
    ref = F.relu(F.conv2d(x.float(), w.float(), padding=3) * scale[None, :, None, None] + bias[None, :, None, None])
    outs = []
    for persistent in (0, ctas):
        out = torch.full((batch, H, W, 24), 5.0, dtype=torch.float16)          # channel pitch 24: 8 foreign channels per pixel
        cpu_hires.cpu_stem(p(x_nhwc), p(w_k), p(scale), p(bias), p(out), batch, H, W, 24, 1, persistent)
        assert float((out[..., 16:] - 5.0).abs().max()) == 0.0
        outs.append(out[..., :16].clone())
    err = float((outs[0].permute(0, 3, 1, 2).float() - ref).abs().max() / ref.abs().max())
    assert err <= 2e-3, "emulated per-tile stem vs torch: %g" % err
    assert torch.equal(outs[0], outs[1])
    # ---- level0 on the stem's output (input pitch 24, output pitch 16)
    w0 = (torch.randn(16, 16, 3, 3, generator=g) / 12.).half()
    x0 = torch.full((batch, H, W, 24), 7.0, dtype=torch.float16)
    x0[..., :16] = outs[0]
    ref0 = F.conv2d(outs[0].permute(0, 3, 1, 2).float(), w0.float(), padding=1) * scale[None, :, None, None] + bias[None, :, None, None]
    res, w0_k = [], w0.permute(0, 2, 3, 1).contiguous()
    for persistent in (0, ctas):
        out = torch.zeros((batch, H, W, 16), dtype=torch.float16)
        cpu_hires.cpu_conv3x3_c16(p(x0), p(w0_k), p(scale), p(bias), p(out), batch, H, W, 24, 16, 0, persistent)
        res.append(out)
    err = float((res[0].permute(0, 3, 1, 2).float() - ref0).abs().max() / ref0.abs().max())
    assert err <= 2e-3, "emulated per-tile level0 vs torch: %g" % err
    assert torch.equal(res[0], res[1])


@pytest.mark.parametrize("cin,cout,H,W,batch,ctas", [(16, 32, 36, 140, 1, 2), (32, 64, 20, 200, 2, 3)])
def test_persistent_stride2_hires_kernels_reproduce_the_per_tile_kernels(cpu_hires, cin, cout, H, W, batch, ctas):
    """level1 (16 -> 32) / level2.tree1.conv1 (32 -> 64), 3x3 stride 2: persistent forms (weights as register-resident B fragments,
    for 64 output channels two warps per row, ragged tiles, several tiles per CTA) against the per-tile kernel -- bit for bit --
    and both against torch."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(cin + H)
    x = torch.randn(batch, cin, H, W, generator=g).half()
    w = (torch.randn(cout, cin, 3, 3, generator=g) / (3. * cin ** 0.5)).half()
    scale, bias = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    ld_in, ld_out = cin + 8, cout + 16
    x_nhwc = torch.full((batch, H, W, ld_in), 3.0, dtype=torch.float16)
    x_nhwc[..., :cin] = x.permute(0, 2, 3, 1)
    w_k = w.permute(0, 2, 3, 1).contiguous()
    ref = F.relu(F.conv2d(x.float(), w.float(), stride=2, padding=1) * scale[None, :, None, None] + bias[None, :, None, None])
    outs = []
    for persistent in (0, ctas):
        out = torch.full((batch, H // 2, W // 2, ld_out), 5.0, dtype=torch.float16)
        cpu_hires.cpu_conv3x3_s2(p(x_nhwc), p(w_k), p(scale), p(bias), p(out), batch, H, W, cin, ld_in, ld_out, 1, persistent)
        assert float((out[..., cout:] - 5.0).abs().max()) == 0.0
        outs.append(out[..., :cout].clone())
    err = float((outs[0].permute(0, 3, 1, 2).float() - ref).abs().max() / ref.abs().max())
    assert err <= 2e-3, "emulated per-tile kernel vs torch: %g" % err
    assert torch.equal(outs[0], outs[1])
