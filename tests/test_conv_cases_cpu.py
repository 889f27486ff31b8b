"""The conv edge-case table and its harness (tests/conv_cases.py), without a GPU.

- The table covers every kernel form smot_conv2d can launch, and every case names its branch and its expectation.
- The harness, run over host memory with a stand-in launch (torch on the dtype-rounded operands, accumulated in fp32 and
  rounded to the output dtype), passes every clean case: exact cases bit for bit, gauss cases within the bound.
- Seeded output faults are each flagged by a named case.
"""
import pytest
import torch
import torch.nn.functional as F

import conv_cases as cc
import launch_check as lc

# every kernel form: the 8 wgmma variants and the reduce kernel, both forms of each hires layer, every small-N kernel,
# every SIMT <tile config, vector> form
ALL_FORMS = (["conv_tc_kernel<%d,%d>" % v for v in ((64, 2), (64, 4), (64, 8), (128, 2), (128, 3), (128, 6), (256, 3),
                                                     (256, 4))]
             + ["splitk_reduce_kernel", "stem7x7_hires_kernel", "stem7x7_persist_kernel", "conv3x3_hires_kernel<16,16,1>",
                "conv3x3_c16_persist_kernel", "conv3x3_hires_kernel<16,32,2>", "conv3x3_s2_persist_kernel<16,32>",
                "conv3x3_hires_kernel<32,64,2>", "conv3x3_s2_persist_kernel<32,64>",
                "conv_smalln_mma_kernel<half,1>", "conv_smalln_mma_kernel<half,2>", "conv_smalln_mma_kernel<float,2>"]
             + ["conv_smalln_direct_kernel<float,float,%d>" % c for c in (4, 8, 16)]
             + ["conv_smalln_kernel<float,float,%d>" % c for c in (4, 8, 16)]
             + ["conv_simt_kernel<float,float,%s,%d>" % (cfg, v) for cfg in ("64,64,4,4", "128,64,8,4", "256,16,4,4")
                for v in (0, 1)])


def test_table_covers_every_kernel_form():
    launched = {k for c in cc.CASES for k in c.kernels}
    missing = [k for k in ALL_FORMS if k not in launched]
    assert not missing, "no case launches %s" % missing
    assert {c.wk for c in cc.CASES if c.wk} == {1, 2, 4, 8}, "every K slicing of the small-N mma kernel"
    assert {c.splits for c in cc.CASES if c.splits} >= {1, 3, 4, 5, 6, 7, 8}, "every default split factor"
    for dt, odt in ((torch.float32, torch.float32), (torch.float16, torch.float16), (torch.float16, torch.float32)):
        forms = {k for c in cc.CASES if c.family == "simt" and (c.dt, c.odt) == (dt, odt) for k in c.kernels}
        assert len(forms) == 6, "all six SIMT forms in %s -> %s: %s" % (dt, odt, sorted(forms))


def test_every_case_names_its_branch():
    for c in cc.CASES:
        assert c.why and c.kernels and c.family in ("wgmma", "hires", "smalln", "simt"), c.name
    for spec in cc.child_cases().values():
        for name, _ in spec["cases"]:
            assert name in cc.BY_NAME


def test_kernel_ids_from_profiler_names():
    assert cc.kernel_id("void smot::conv_tc_kernel<(int)128, (int)2>(CUtensorMap_st, CUtensorMap_st, smot::TcArgs)") == \
        "conv_tc_kernel<128,2>"
    assert cc.kernel_id("void smot::conv_tc_kernel<128, 2>(CUtensorMap_st, CUtensorMap_st, smot::TcArgs)") == \
        "conv_tc_kernel<128,2>"
    assert cc.kernel_id("void smot::conv_simt_kernel<__half, float, 256, 16, 4, 4, true>(smot::ConvArgs)") == \
        "conv_simt_kernel<half,float,256,16,4,4,1>"
    assert cc.kernel_id("smot::splitk_reduce_kernel(smot::TcArgs)") == "splitk_reduce_kernel"
    assert cc.kernel_id("void at::native::vectorized_elementwise_kernel<4>(int)") is None


# ---- the harness over host memory --------------------------------------------------------------------------------------
def standin(p, fault=None):
    """The convolution of p.d computed by torch over host memory: fp32 accumulation of the dtype-rounded operands, the
    epilogue in fp32, rounded to the output dtype.  `fault` seeds one output fault (see FAULTS)."""
    d, case = p.d, p.case
    mem = lc.Memory("cpu")
    x, w, s, b, res = lc.conv_snapshot(mem, d)
    if fault == "residual-pitch":
        res = mem.nhwc(d.residual, d.batch, d.OH, d.OW, d.Cout, d.out_ld, case.dt).double()
    xc, wc = x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2)
    acc = F.conv2d(xc, wc, None, d.stride, d.pad)
    K = d.KH * d.KW * d.Cin
    if fault in ("last-split-dropped", "last-split-twice"):
        # the K range of the last split (K index = tap * Cin + channel, 64 per chunk)
        chunks = K // 64
        cps = -(-chunks // case.splits)
        wl = torch.zeros_like(wc).permute(0, 2, 3, 1).reshape(d.Cout, K)
        wl[:, 64 * cps * (case.splits - 1):] = w.float().reshape(d.Cout, K)[:, 64 * cps * (case.splits - 1):]
        part = F.conv2d(xc, wl.reshape(d.Cout, d.KH, d.KW, d.Cin).permute(0, 3, 1, 2), None, d.stride, d.pad)
        acc = acc - part if fault == "last-split-dropped" else acc + part
    if fault == "s2-tap-off":
        # tap (0, 0) read one input column to the right
        w0 = torch.zeros_like(wc)
        w0[:, :, 0, 0] = wc[:, :, 0, 0]
        xs = torch.zeros_like(xc)
        xs[..., :-1] = xc[..., 1:]
        acc = acc - F.conv2d(xc, w0, None, d.stride, d.pad) + F.conv2d(xs, w0, None, d.stride, d.pad)
    y = acc
    if s is not None:
        y = y * s.float().view(1, -1, 1, 1)
    if b is not None:
        y = y + b.float().view(1, -1, 1, 1)
    if res is not None:
        y = y + res.float().permute(0, 3, 1, 2)
    if d.relu:
        y = y.clamp_min(0.0)
    y = y.permute(0, 2, 3, 1).to(case.odt)
    if fault == "row-shift":
        y[:, -1, 1:] = y[:, -1, :-1].clone()
    if fault == "n-tile-offset":
        y[..., 64:128] = y[..., 0:64].clone()
    if fault == "next-image":
        y[1, 0] = y[0, -1]
    out = mem.nhwc(d.out, d.batch, d.OH, d.OW, d.Cout, d.out_ld, case.odt)
    out.copy_(y)
    if fault == "pitch-gap":
        mem.view(d.out + d.Cout * out.element_size(), (1,), None, case.odt).fill_(0.0)


# seeded output fault -> the case that must flag it
FAULTS = {
    "row-shift": "tile-ragged-batch",              # a tile row shifted by one pixel at the ragged bottom edge
    "last-split-dropped": "split-4-ragged",        # the last split's K range (chunks 15..17) missing
    "last-split-twice": "split-empty-rounding",    # the last split's K range (chunks 30..32) counted twice
    "n-tile-offset": "bn-95-tiles",                # the second 64-channel N tile written at the first tile's offset
    "residual-pitch": "tile-ragged-batch",         # the residual read with out_ld (144) as its pitch (res_ld 160)
    "s2-tap-off": "s2-ow-odd",                     # a stride-2 tap one input pixel off
    "pitch-gap": "ld-8mod64",                      # a write into the output's pitch gap
    "next-image": "s2-batch-straddle",             # image 0's last row written over the next image's first row
}

# The host reference costs about 4 float64 MACs per MAC of the case: the few largest cases of the table run in the GPU
# module only.
HOST_MACS = 3e8


def _host_cases():
    return [c for c in cc.CASES if c.macs() <= HOST_MACS]


def test_most_of_the_table_runs_on_the_host():
    assert len(_host_cases()) >= 0.8 * len(cc.CASES)


@pytest.mark.parametrize("pattern", ["exact", "gauss"])
def test_harness_passes_clean_results(pattern):
    worst = 0.0
    for case in _host_cases():
        r = cc.run_case(case, pattern, "cpu", standin)
        assert r.ok, r.describe()
        worst = max(worst, r.max_ratio)
    print("%s: %d cases clean, worst |err|/bound %.3f" % (pattern, len(_host_cases()), worst))


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_harness_flags_seeded_fault(fault):
    case = cc.BY_NAME[FAULTS[fault]]
    for pattern in ("exact", "gauss"):
        r = cc.run_case(case, pattern, "cpu", lambda p: standin(p, fault))
        print("%s on %s/%s: %s" % (fault, case.name, pattern, r.describe()))
        if fault == "pitch-gap":
            assert r.guards, "%s not flagged" % fault
        else:
            assert not r.ok, "%s not flagged by %s/%s" % (fault, case.name, pattern)
            if pattern == "exact":
                assert r.exact_ok is False
