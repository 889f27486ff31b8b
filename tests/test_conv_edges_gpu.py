"""smot_conv2d at its tile, ring, split-K, pitch and batch edges, on every kernel form (cases: tests/conv_cases.py).

Each case runs with both operand patterns: "exact" must equal the float64 reference bit for bit, "gauss" must meet the
per-element bound of tests/launch_check.py.  Both must leave the memory around the output, the input, the residual and the
workspace's reserved counter bytes untouched.  The exact run is recorded with torch.profiler, and the kernels it launched
(and the split factor / small-N K slicing read from their grids) must be the case's expectation, so that a routing change
fails here instead of quietly testing another kernel.

Bit invariance across batching, found on the H100 for every form the batched plans use: the wgmma kernel without and with
split-K (the split factor is chosen per image), the small-N mma kernel (WK chosen per image), the small-N direct and
shared-memory kernels, the SIMT kernel and the hires per-tile and persistent kernels each give a batch-B output equal bit
for bit to B batch-1 calls.
"""
import copy
import json
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import conv_cases as cc

pytestmark = pytest.mark.gpu
RESULTS = {}
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def _sm_ok():
    # the kernel expectations hold from 120 to 144 SMs (see conv_cases)
    return 120 <= torch.cuda.get_device_properties(0).multi_processor_count <= 144


def _launch_recorded(case, launched):
    def launch(p):
        assert cc.gpu_algo(p) == case.algo, "%s: smot_conv2d_algo %d, expected %d" % (case.name, cc.gpu_algo(p), case.algo)
        launched.extend(cc.profiled(lambda: cc.gpu_launch(p)))
    return launch


@pytest.mark.parametrize("case", cc.CASES, ids=lambda c: c.name)
def test_conv_edge_case(case, monkeypatch):
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    for pattern in ("exact", "gauss"):
        launched = []
        r = cc.run_case(case, pattern, "cuda", _launch_recorded(case, launched) if pattern == "exact" else cc.gpu_launch)
        RESULTS[(case.name, pattern)] = r
        assert r.ok, r.describe()
        if pattern == "exact" and _sm_ok():
            assert [k for k, _ in launched] == list(case.kernels), "%s (%s) launched %s" % (case.name, case.why, launched)
            errs = cc.expected_grid_check(case, launched)
            assert not errs, "%s: %s" % (case.name, errs)


def _variant(case, **kw):
    c = copy.copy(case)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _output(case, ops, env=None, monkeypatch=None):
    if env:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
    r = cc.run_case(case, "gauss", "cuda", cc.gpu_launch, ops=ops, keep_output=True)
    assert r.ok, r.describe()
    if env:
        for k in env:
            monkeypatch.delenv(k)
    return r.output


# form -> (case, batch): a batch size that keeps the case on its route
BATCHED = {"wgmma": ("tile-ragged-batch", 3), "wgmma-split": ("split-8-level5", 2), "smalln-mma": ("sn-mma-c9-wk8", 3),
           "smalln-direct": ("sn-direct-batch2", 3), "smalln-smem": ("sn-smem-1025", 2), "simt": ("simt-vec-f16-f16", 3),
           "hires-per-tile": ("hires-c16-per-tile", 3), "hires-persistent": ("hires-s2-32-64-persistent", 3),
           "hires-stem": ("stem-odd-w", 2)}


@pytest.mark.parametrize("form", sorted(BATCHED))
def test_batched_pass_equals_per_image_passes(form, monkeypatch):
    name, B = BATCHED[form]
    base = cc.BY_NAME[name]
    for k, v in base.env.items():
        monkeypatch.setenv(k, v)
    case = _variant(base, B=B, name=name + "-b%d" % B)
    ops = cc.make_operands(case, "gauss", "cuda")
    whole = _output(case, ops)
    one = _variant(base, B=1, name=name + "-b1")
    for b in range(B):
        part = {k: (v[b:b + 1] if k in ("x", "res") and v is not None else v) for k, v in ops.items()}
        assert torch.equal(_output(one, part), whole[b:b + 1]), "%s: image %d of the batch-%d pass differs" % (form, b, B)


@pytest.mark.parametrize("name,depths", [("ring-bn64-st4-k9", ("2", "4", "8")), ("ring-bn128-st6-k13", ("2", "3", "6")),
                                         ("ring-bn256-st4-k9", ("3", "4"))])
def test_ring_depths_give_the_same_bits(name, depths, monkeypatch):
    case = _variant(cc.BY_NAME[name], env={})
    ops = cc.make_operands(case, "gauss", "cuda")
    outs = [_output(case, ops, {"SMOT_TC_STAGES": d}, monkeypatch) for d in depths]
    for d, o in zip(depths[1:], outs[1:]):
        assert torch.equal(o, outs[0]), "%s: ring depth %s differs from depth %s" % (name, d, depths[0])


@pytest.mark.parametrize("name", ["split-8-level5", "split-batch10-2stage", "split-empty-rounding", "fc6-30"])
def test_k_slices_equal_split_k(name, monkeypatch):
    case = cc.BY_NAME[name]
    ops = cc.make_operands(case, "gauss", "cuda")
    split = _output(case, ops)
    sliced = _output(case, ops, {"SMOT_TC_SLICED": "1"}, monkeypatch)
    assert torch.equal(sliced, split)


@pytest.mark.parametrize("layer", ["stem", "c16", "s2-16-32", "s2-32-64"])
def test_hires_persistent_equals_per_tile(layer, monkeypatch):
    tile, pers = cc.BY_NAME["hires-%s-per-tile" % layer], cc.BY_NAME["hires-%s-persistent" % layer]
    ops = cc.make_operands(tile, "gauss", "cuda")
    a = _output(_variant(tile, env={}), ops, tile.env, monkeypatch)
    b = _output(_variant(pers, env={}), ops, pers.env, monkeypatch)
    assert torch.equal(a, b)


@pytest.mark.parametrize("layer", ["stem", "c16", "s2-16-32", "s2-32-64"])
def test_persistent_loop_equals_per_tile(layer, monkeypatch):
    """More tiles than CTAs: every CTA after its first tile runs the prefetched one, bit for bit the per-tile kernel's."""
    case = cc.BY_NAME["hires-%s-persistent-loop" % layer]
    ops = cc.make_operands(case, "gauss", "cuda")
    a = _output(case, ops)
    b = _output(case, ops, {"SMOT_HIRES_PERSIST": "0"}, monkeypatch)
    assert torch.equal(a, b)


# ---- switches held in statics: one child process per environment ------------------------------------------------------
_CHILD = r"""
import json, os, sys
sys.path[:0] = json.loads(sys.argv[1])
import torch
import conv_cases as cc
spec, out = json.loads(sys.argv[2]), sys.argv[3]
res = []
for name, env in spec:
    case = cc.BY_NAME[name]
    env = dict(case.env, **(env or {}))
    os.environ.update(env)
    for pattern in ("exact", "gauss"):
        launched = []
        r = cc.run_case(case, pattern, "cuda", lambda p: launched.extend(cc.profiled(lambda: cc.gpu_launch(p))),
                        keep_output=True)
        res.append(dict(name=name, env=env, pattern=pattern, output=r.output, ok=r.ok, describe=r.describe(),
                        kernels=launched))
    for k in env:
        del os.environ[k]
torch.save(res, out)
"""


def _child(env, spec):
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "out.pt")
        e = dict(os.environ)
        for k in ("SMOT_TC_CLUSTER", "SMOT_TC_MAXSPLIT", "SMOT_TC_NOSPLIT", "SMOT_TC_MINCTAS", "SMOT_TC_STAGES",
                  "SMOT_TC_SLICED"):
            e.pop(k, None)
        e.update(env)
        p = subprocess.run([sys.executable, "-c", _CHILD, json.dumps([HERE, REPO]), json.dumps(spec), out], env=e,
                           capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, "child process failed:\n%s\n%s" % (p.stdout[-3000:], p.stderr[-3000:])
        return torch.load(out, weights_only=False)


# (case, SMOT_TC_STAGES) -> the only launch with SMOT_TC_CLUSTER=1: (kernel, grid.z).  On an H100 SXM the clusters of these
# variants all fit at once (cudaOccupancyMaxActiveClusters), so the cluster finish is taken, on the 3 / 4-stage ring.
CLUSTER_2STAGE_ROUTES = {("split-8-level5", "2"): ("conv_tc_kernel<128,3>", 8),
                         ("split-batch10-2stage", None): ("conv_tc_kernel<64,4>", 4)}


def test_cluster_finish_equals_reduce_kernel(monkeypatch):
    """SMOT_TC_CLUSTER=1: the split CTAs of a tile finish it inside their cluster.  Bit for bit the reduce path, including
    the two routes to a 2-stage ring (forced by SMOT_TC_STAGES=2, and batch 10 of 3x3 256 -> 64 at 44x80), which launch
    the 3 / 4-stage kernel of the same N tile instead: the 2-stage kernels carry no cluster finish."""
    spec = cc.child_cases()["cluster"]
    got = _child(spec["env"], spec["cases"])
    finished_in_cluster, bad = [], []
    for rec in got:
        what = "%s/%s %s" % (rec["name"], rec["pattern"], rec["env"])
        if not rec["ok"]:
            bad.append("SMOT_TC_CLUSTER=1 %s: %s" % (what, rec["describe"]))
            continue
        case = cc.BY_NAME[rec["name"]]
        for k, v in rec["env"].items():
            monkeypatch.setenv(k, v)
        ref = cc.run_case(case, rec["pattern"], "cuda", cc.gpu_launch, keep_output=True)
        for k in rec["env"]:
            monkeypatch.delenv(k)
        if not torch.equal(rec["output"], ref.output):
            bad.append("%s: the cluster finish differs from the reduce kernel" % what)
        names = [k for k, _ in rec["kernels"]]
        if "splitk_reduce_kernel" not in names:
            if any(n.startswith("conv_tc_kernel<") and n.endswith(",2>") for n in names):
                bad.append("%s: a 2-stage kernel without the reduce kernel: %s" % (what, names))
            finished_in_cluster.append("%s %s" % (what, names))
        # the two 2-stage routes: the lifted ring, the whole split in one cluster launch, no reduce kernel
        want = CLUSTER_2STAGE_ROUTES.get((rec["name"], rec["env"].get("SMOT_TC_STAGES")))
        if want is not None and _sm_ok() and [(k, g[2]) for k, g in rec["kernels"]] != [want]:
            bad.append("%s: launched %s, expected only %s with %d K splits" % (what, rec["kernels"], want[0], want[1]))
    print("finished inside the cluster:\n  " + "\n  ".join(finished_in_cluster))
    assert not bad, "\n".join(bad)
    assert finished_in_cluster, "no case took the cluster finish"


def test_maxsplit2_split_factor():
    """SMOT_TC_MAXSPLIT=2: the split factor 2, which the default rule never produces."""
    spec = cc.child_cases()["maxsplit2"]
    for rec in _child(spec["env"], spec["cases"]):
        assert rec["ok"], rec["describe"]
        tc = [g for k, g in rec["kernels"] if k.startswith("conv_tc_kernel")]
        assert tc and tc[0][2] == 2 and rec["kernels"][-1][0] == "splitk_reduce_kernel", rec["kernels"]


def test_zz_summary():
    """Per kernel family: the cases run in this session, the worst gauss |err|/bound, and that every exact run was
    bit-exact."""
    if not RESULTS:
        pytest.skip("no case ran in this session")
    fams = {}
    for (name, pattern), r in RESULTS.items():
        f = fams.setdefault(r.case.family, dict(cases=set(), worst=0.0, exact=0, exact_ok=0))
        f["cases"].add(name)
        if pattern == "gauss":
            f["worst"] = max(f["worst"], r.max_ratio)
        else:
            f["exact"] += 1
            f["exact_ok"] += int(bool(r.exact_ok))
    for fam, f in sorted(fams.items()):
        print("%-7s %3d cases, worst gauss |err|/bound %.3f, exact runs bit for bit: %d of %d"
              % (fam, len(f["cases"]), f["worst"], f["exact_ok"], f["exact"]))
        assert f["exact_ok"] == f["exact"]
