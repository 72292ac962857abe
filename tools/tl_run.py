"""Development aid: build the -DIAF_TC_TIMELINE variant of the library (iaf_b200/lib/libiaf_tl.so, rebuilt when a
source is newer), run one IAF step of a bench.py workload and print the in-kernel timeline of CTA 0 (see TL() in
iaf_b200/csrc/iaf_tc.cu), then the cycles of every phase per tile and the producer's ring waits.

    python tools/tl_run.py [workload] [stage]

stage: which launch of a per-stage step records (IAF_TL_STAGE; default the last).  A one-launch step always records.
"""
import ctypes
import io
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import iaf_b200.build as B  # noqa: E402

B.LIB = B.build(lib=os.path.join(B.LIBDIR, "libiaf_tl.so"), defines=["IAF_TC_TIMELINE"])
import iaf_b200._lib as L  # noqa: E402

L.LIB = B.LIB
import torch  # noqa: E402
from bench import make_workload  # noqa: E402

PHASE = {15: "MMA operands ready", 20: "MMAs done", 21: "acc tile written", 35: "heads operands ready",
         40: "heads MMAs done", 41: "heads acc written", 10: "window built", 25: "acc ready", 30: "(hidden) epilogue done",
         45: "heads acc ready", 50: "heads epilogue done", 99: "end"}
ROLE = {0: "MMA warpgroups", 1: "epilogue warps"}


def run(name, stage):
    if stage is not None:
        os.environ["IAF_TL_STAGE"] = str(stage)
    dev = torch.device("cuda:0")
    op, layers, sets = make_workload(name, dev, 2)
    s = sets[0]
    for _ in range(3):
        op.step(s["z"], s["ctx"])
    torch.cuda.synchronize()
    lib = ctypes.CDLL(B.LIB)
    lib.iaf_tc_timeline_dump()  # discard warm-up events
    op.step(s["z"], s["ctx"])
    torch.cuda.synchronize()
    # the dump prints from C: capture file descriptor 1
    sys.stdout.flush()
    r, w = os.pipe()
    saved = os.dup(1)
    os.dup2(w, 1)
    lib.iaf_tc_timeline_dump()
    ctypes.CDLL(None).fflush(None)
    os.dup2(saved, 1)
    os.close(w)
    with io.open(r) as f:
        text = f.read()
    ev = []
    for line in text.splitlines():
        if line.startswith("TL"):
            d = dict(x.split("=") for x in line.split()[1:])
            ev.append((int(d["t"]), int(d["role"]), int(d["tag"]), int(d["k"])))
    ev.sort()
    print("=== %s, stage %s: %d events ===" % (name, "last" if stage is None else stage, len(ev)))
    for t, role, tag, k in ev:
        print("%9d  role%d  %-24s k=%d" % (t, role, PHASE.get(tag, {60: "ring wait", 61: "ring released"}.get(tag, tag)), k))
    # phase cycles per role: its events are phase ends, in order; each phase lasts from the previous event to its own.
    # The two roles run concurrently, so their phases of neighbouring tiles overlap in time (compare the t column).
    for role in (0, 1):
        w = [e for e in ev if e[1] == role]
        print("--- %s: cycles per phase (lane 0 of its first warp) ---" % ROLE[role])
        for (t0, _, g0, k0), (t1, _, g1, k1) in zip(w, w[1:]):
            print("tile %d  %-24s -> %-24s %7d  (ends at %d)" % (k1 if g1 != 99 else k0, PHASE.get(g0), PHASE.get(g1),
                                                                t1 - t0, t1))
    waits = [(e[0], e[2], e[3]) for e in ev if e[1] == 2]
    tot = sum(b[0] - a[0] for a, b in zip(waits, waits[1:]) if a[1] == 60 and b[1] == 61)
    if waits:
        print("--- producer: %d ring waits, %d cycles waiting in all ---" % (sum(1 for x in waits if x[1] == 60), tot))


if __name__ == "__main__":
    name = sys.argv[1] if len(sys.argv) > 1 else "c2a"
    run(name, int(sys.argv[2]) if len(sys.argv) > 2 else None)
