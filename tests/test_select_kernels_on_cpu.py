"""The source text of the proposal-selection kernels and of their entry points (csrc/select_nms.cu: sort + NMS in both
instantiations, the segment scatter, the three RPN kernels) compiled for the host over tests/cpu_cuda/shim_warp.h and run on
the edge tables of tests/select_cases.py at reduced sizes: n_max <= 1186 (both reduce paths), RPN levels of one chunk, one
chunk + 3 anchors, 1x1 and 21 chunks.  The kernels are validated on the GPU (test_select_edges_gpu.py), so this run
reproducing the references validates the shim's warp collectives; seeded mutants -- textual substitutions of the source --
show that the tables catch faults at the edges they target."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest
import torch

import select_cases as sc

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "cpu_cuda"))

N_CPU = (1, 63, 64, 65, 129)
N_CPU_LARGE = (1185, 1186)          # the last staged and the first global-memory bitmask: the scene thresholds, max_keep = all
SEGMENTED_CPU = [(1, 2, 64), (3, 3, 65), (3, 9, 64), (1, 2, 1186)]
RPN_CPU = ("one-chunk-distinct", "chunk+3-straddle", "pm-zero", "pm-zero-top1", "saturated-extreme", "level-ties-min-size",
           "top1-ties", "21-chunks-all-equal")
CPU_MAX_KEEPS = lambda kept: sorted({0, 1, 65, max(kept - 1, 0), kept})   # noqa: E731

# each mutant: the substitutions, then the table that targets it first (the others follow)
MUTANTS = {
    "iou_ge": ("iou_plus1(bi, bj) > a.thresh", "iou_plus1(bi, bj) >= a.thresh"),
    "tie_key": ("| (unsigned long long)(0xFFFFFFFFu - (unsigned)i);", "| (unsigned long long)((unsigned)i);",
                "const unsigned idx = 0xFFFFFFFFu - (unsigned)(keys[i] & 0xFFFFFFFFull);",
                "const unsigned idx = (unsigned)(keys[i] & 0xFFFFFFFFull);"),
    "cache_copy": ("if (w > (row >> 6)) cache", "if (w > (row >> 6) + 1) cache"),
    "max_keep_drops_lowest": ("kept &= ~(1ull << (63 - __clzll((long long)kept)));", "kept &= kept - 1ull;"),
    "radix_pick_gt": ("if (key != 0ull && key >= T) {", "if (key != 0ull && key > T) {"),
    "level_tie": ("if (o < l ? v >= s : v > s)", "if (v > s)"),
    "scatter_prefix": ("base += q < cls ? c : 0;", "base += q <= cls ? c : 0;"),
}


@pytest.fixture(scope="module")
def builds(tmp_path_factory):
    """The unmodified build and every mutant, compiled concurrently."""
    import cpu_cuda_build as cpu_build
    d = tmp_path_factory.mktemp("select_cpu")
    jobs = {"base": None, **MUTANTS}
    with ThreadPoolExecutor(max_workers=len(jobs)) as pool:
        futs = {k: pool.submit(cpu_build.build_select, str(d / ("_select_%s.so" % k)), m) for k, m in jobs.items()}
        return {k: f.result() for k, f in futs.items()}


@pytest.fixture(scope="module")
def cpu_ops(builds):
    return sc.CpuOps(builds["base"])


def _rpn_specs():
    specs = {s["name"]: s for s in sc.rpn_cases()}
    return [specs[n] for n in RPN_CPU]


def rpn_table(ops_, stop_at_first=False):
    """Single-image and batched (B = 3, the first three single-image specs' tie structures on one shape) RPN runs."""
    calls, failures, worst = 0, [], (0.0, 0.0)
    for spec in _rpn_specs():
        logits_l, deltas_l, heads = sc.rpn_image(spec, 77)
        ref = sc.rpn_case_reference(spec, logits_l, deltas_l)
        ob, os_, oc = sc.run_rpn(ops_, "cpu", spec, heads)
        calls += 1
        err, ws, wb = sc.check_rpn(spec, ob[0], os_[0], int(oc[0]), ref)
        worst = (max(worst[0], ws), max(worst[1], wb))
        if err:
            failures.append((spec["name"], err))
            if stop_at_first:
                return calls, failures, worst
    shapes = [(15, 239), (1, 1)]
    specs, refs, heads = [], [], []
    for b, kind in enumerate(("straddle", "pm_zero", "level_ties")):
        spec = dict(name="batched/%d" % b, levels=[s + (kind,) for s in shapes], pre=1000, post=500, fpn=700, nms=0.7,
                    amodal=False, img=(333, 517))
        logits_l, deltas_l, h = sc.rpn_image(spec, 90 + b)
        specs.append(spec)
        refs.append(sc.rpn_case_reference(spec, logits_l, deltas_l))
        heads.append(h)
    cat = [torch.cat([h[lv] for h in heads]) for lv in range(len(shapes))]
    ob, os_, oc = sc.run_rpn(ops_, "cpu", specs[0], cat, batched=True)
    calls += 1
    for b in range(3):
        err, ws, wb = sc.check_rpn(specs[b], ob[b], os_[b], int(oc[b]), refs[b])
        worst = (max(worst[0], ws), max(worst[1], wb))
        if err:
            failures.append((specs[b]["name"], err))
    return calls, failures, worst


def sort_nms_cpu_table(ops_, stop_at_first=False):
    calls, failures = sc.sort_nms_table(ops_, "cpu", N_CPU, extra=(0.0,), max_keeps=CPU_MAX_KEEPS, stop_at_first=stop_at_first)
    if failures and stop_at_first:
        return calls, failures
    c, f = sc.sort_nms_table(ops_, "cpu", N_CPU_LARGE, extra=(), max_keeps=lambda kept: [kept], stop_at_first=stop_at_first)
    return calls + c, failures + f


def test_sort_nms_source_on_cpu(cpu_ops):
    before = cpu_ops.launches()
    calls, failures = sort_nms_cpu_table(cpu_ops)
    assert not failures, failures[:5]
    assert calls > 300 and cpu_ops.launches() > before


def test_sort_nms_segmented_source_on_cpu(cpu_ops):
    calls, failures = sc.segmented_table(cpu_ops, "cpu", SEGMENTED_CPU)
    assert not failures, failures[:5]


def test_sort_nms_segmented_refusal_launches_nothing(cpu_ops):
    batch, ncls = 65536, 2
    before = cpu_ops.launches()
    with pytest.raises(RuntimeError, match="65536 segments"):
        cpu_ops.sort_nms_segmented(torch.zeros(batch, ncls, 4), torch.ones(batch, ncls), torch.ones(batch, dtype=torch.int32),
                                   batch, ncls, 0.0, 0.5, 1, torch.zeros(batch, 1, 4), torch.zeros(batch, 1),
                                   torch.zeros(batch, 2, dtype=torch.int32))
    assert cpu_ops.launches() == before


def test_rpn_select_source_on_cpu(cpu_ops):
    calls, failures, worst = rpn_table(cpu_ops)
    assert not failures, failures
    assert worst[0] <= 1.0 and worst[1] <= 1.0


MUTANT_FIRST_TABLE = {"radix_pick_gt": "rpn_select", "level_tie": "rpn_select", "scatter_prefix": "sort_nms_segmented"}


def first_failure(path, first="sort_nms"):
    """The first table case the build at `path` fails: (table, case) or None.  The table `first` runs first; each table's
    name is printed as it starts."""
    ops_ = sc.CpuOps(path)
    tables = [("sort_nms", lambda: sort_nms_cpu_table(ops_, stop_at_first=True)[1]),
              ("sort_nms_segmented", lambda: sc.segmented_table(ops_, "cpu", SEGMENTED_CPU, stop_at_first=True)[1]),
              ("rpn_select", lambda: rpn_table(ops_, stop_at_first=True)[1])]
    tables.sort(key=lambda t: t[0] != first)
    for name, run in tables:
        print("TABLE", name, flush=True)
        f = run()
        if f:
            return name, f[0]
    return None


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_seeded_mutant_is_caught(builds, mutant):
    """Each mutant runs in a child process: a mutant may also read out of bounds (e.g. a radix select that returns fewer
    than k keys leaves empty slots that decode to anchor 2^22 - 1), which ends the child with a signal -- also a catch."""
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_select_kernels_on_cpu as t; print('CAUGHT', t.first_failure(%r, %r))"
            % (os.path.dirname(HERE), HERE, builds[mutant], MUTANT_FIRST_TABLE.get(mutant, "sort_nms")))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       cwd=os.path.dirname(HERE))
    lines = r.stdout.splitlines()
    if r.returncode < 0:
        table = [ln for ln in lines if ln.startswith("TABLE")][-1]
        caught = "%s: terminated by signal %d" % (table, -r.returncode)
    else:
        assert r.returncode == 0, r.stdout[-3000:]
        caught = [ln for ln in lines if ln.startswith("CAUGHT")][-1]
        assert caught != "CAUGHT None", "mutant %s passes every table" % mutant
    print("\nmutant %s: %s" % (mutant, caught))
