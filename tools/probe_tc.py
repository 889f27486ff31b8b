"""Developer tool: phase timestamps (ns, %globaltimer) of CTA 0 of one wgmma conv launch."""
import math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
dbg = torch.zeros(136, dtype=torch.int64, device="cuda")
os.environ["SMOT_TC_DEBUG"] = hex(dbg.data_ptr())
from siammot_b200 import ops
dt = torch.float16
for name, B, Cin, H, W, Cout, k in [("level5 3x3", 1, 512, 22, 40, 512, 3), ("level3 3x3", 1, 128, 88, 160, 128, 3), ("root 1x1 K1280", 1, 1280, 22, 40, 512, 1), ("rpn P2", 1, 128, 176, 320, 128, 3), ("level4 3x3", 1, 256, 44, 80, 256, 3)]:
    x = torch.randn(B, H, W, Cin, device="cuda").to(dt)
    w = (torch.randn(Cout, k, k, Cin, device="cuda") / math.sqrt(Cin * k * k)).to(dt)
    sc = torch.rand(Cout, device="cuda"); bi = torch.randn(Cout, device="cuda")
    out = torch.empty(B, H, W, Cout, device="cuda", dtype=dt)
    for i in range(5):
        dbg.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); ops.conv2d(x, w, sc, bi, None, 1, k // 2, True, out=out); e1.record()
        torch.cuda.synchronize()
    t = dbg.cpu().tolist()
    if os.environ.get("PROBE_ITERS"):
        base = t[0]
        print("  it: producer-ready, tma-issued, mma-data-ready, mma-issued (ns from kernel start)")
        for it in range(0, 20):
            print("  %2d: %6d %6d %6d %6d" % (it, t[40 + it] - base, t[72 + it] - base, t[8 + it] - base, t[104 + it] - base))
    print(name, "events %.1f us |" % (e0.elapsed_time(e1) * 1e3), "prologue %.2f  first-data %.2f  mainloop %.2f  epilogue %.2f  teardown %.2f (us)" % (
        (t[1] - t[0]) / 1e3, (t[2] - t[1]) / 1e3, (t[3] - t[2]) / 1e3, (t[4] - t[3]) / 1e3, (t[5] - t[4]) / 1e3))
