"""Debug aid (GPU box, P2M_TRACE=1 build): event timeline of CTA 0 of the conv kernel of ONE layer of the eval forward
at the bench workload, and per-role busy / wait totals over the logged window.
Usage: P2M_TRACE_V=12288 P2M_TRACE_UNPOOL=0 [P2M_TRACE_FOUT=128] [P2M_TRACE_NTH=k] python tools/umma_trace_model.py [n_events=400]
P2M_TRACE_NTH picks the k-th (from 0) matching launch of the forward, so that exactly one launch is logged (without it
every matching launch writes into the same buffer)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from pose2mesh_release_b200 import _lib  # noqa: E402
from pose2mesh_release_b200.meshnet import Pose2Mesh  # noqa: E402

n_ev = int(sys.argv[1]) if len(sys.argv) > 1 else 400
graph_L, perm_rev = bench.build_problem("smpl")
torch.manual_seed(123)
model = Pose2Mesh(5, 3, graph_L, joint_set="human36")
model.load_state_dict(bench.randomize_bn_({k: v.clone() for k, v in model.state_dict().items()}))
model = model.cuda().set_precision("fp16x3").eval()
x = torch.randn(256, 17, 5, generator=torch.Generator().manual_seed(1000)).cuda()
lib = _lib.load()
buf = torch.zeros(8 * 512, dtype=torch.int64, device="cuda")
with torch.no_grad():
    model(x)
    h = model._hier.handle(0)
    _lib.check(lib.p2m_debug_set_trace(h, buf.data_ptr()), "set_trace (needs a P2M_TRACE=1 build)")
    model(x)
    torch.cuda.synchronize()
    lib.p2m_debug_set_trace(h, None)
t = buf.cpu().numpy().reshape(8, 512)
names = {0: "producer", 1: "bload", 3: "mma + epilogue", 4: "loader"}
ev_all = []
per_role = {r: [] for r in names}
for role in names:
    for v in t[role]:
        if v:
            e = (int(v) & 0xFFFFFFFFFFFF, role, int(v) >> 48)
            ev_all.append(e)
            per_role[role].append(e)
if not ev_all:
    sys.exit("no events logged: check the P2M_TRACE_* filters and the P2M_TRACE=1 build")
ev_all.sort()
t0 = ev_all[0][0]
pn = {1: "wait_x", 2: "x_ready", 6: "T2 gathered", 7: "blocks emitted", 8: "end barrier"}
mn = {1: "tile start", 2: "main loop done", 4: "wait full slot", 5: "slot full -> 12 MMAs",
      # sub-phases of the 64 x 128 (N = 128) epilogue, MMA warp 0
      20: "epi: accumulator staged", 21: "epi: residual in hand", 22: "epi: outputs computed",
      23: "epi: output stores issued"}
for c, role, ev in ev_all[:n_ev]:
    if role == 0:
        label = pn.get(ev, str(ev))
    elif role == 1:
        label = f"slot free -> load B block {ev - 10}"
    elif role == 3:
        label = mn.get(ev, str(ev))
    else:
        label = "stage free" if ev == 1 else "copies issued"
    print(f"{c - t0:9d}  {names[role]:14s} {label}")


def spans(role, a, b):
    """Sum of (time of event b - time of the event a before it) over the role's log, in cycles."""
    tot, last = 0, None
    for c, _, ev in per_role[role]:
        if ev == a:
            last = c
        elif ev == b and last is not None:
            tot += c - last
            last = None
    return tot


t1 = ev_all[-1][0]
window = max(1, t1 - t0)
rows = [
    ("mma", "wait on a full slot", spans(3, 4, 5)),
    ("mma", "issue (slot full -> next wait)", spans(3, 5, 4) + spans(3, 5, 2)),
    ("mma", "epilogue (main loop done -> next tile)", spans(3, 2, 1)),
    ("producer", "wait on staged rows", spans(0, 1, 2)),
    ("producer", "gather", spans(0, 2, 6)),
    ("producer", "empty-slot wait + stores", spans(0, 6, 7)),
    ("producer", "end barrier", spans(0, 7, 8)),
    ("loader", "wait on a free stage", spans(4, 2, 1)),
]
print(f"\nlogged window: {window} cycles (CTA 0; each role's log holds at most 512 events)")
for role, what, cyc in rows:
    print(f"{role:9s} {what:40s} {cyc:10d} cycles  {100.0 * cyc / window:5.1f} %")

# Per-tile split of the MMA warpgroup's time over the tiles whose main loop and epilogue are both in the log: main loop
# (tile start -> main loop done), then every epilogue step (named after the event that ends it), up to the next tile
# start.
steps, tiles, cur, last = {}, 0, None, None
for c, _, ev in per_role[3]:
    if ev in (4, 5):
        continue
    if ev == 1:
        if cur is not None and last is not None:
            cur["next tile start"] = c - last[0]
            for k, v in cur.items():
                steps[k] = steps.get(k, 0) + v
            tiles += 1
        cur, last = {}, (c, ev)
    elif cur is not None:
        cur["main loop" if ev == 2 else mn.get(ev, str(ev))] = c - last[0]
        last = (c, ev)
if tiles:
    print(f"\nper tile, MMA warp 0, mean over {tiles} tiles (cycles)")
    for k, v in steps.items():
        print(f"  {k:32s} {v / tiles:9.0f}")
    epi = sum(v for k, v in steps.items() if k != "main loop")
    print(f"  {'epilogue total (to next start)':32s} {epi / tiles:9.0f}")
