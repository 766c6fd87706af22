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
# roles 3 and 5: warp 0 of MMA + epilogue warpgroup 0 (every tile, or the even tiles of the 64 x 128 configuration)
# and 1 (its odd tiles)
names = {0: "producer", 1: "bload", 3: "mma wg0", 4: "loader", 5: "mma wg1"}
MMA = (3, 5)
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
mn = {1: "tile start", 3: "turn: previous tile's main loop done", 2: "main loop done", 4: "wait full slot",
      5: "slot full -> MMAs",
      # sub-phases of the 64 x 128 (N = 128) epilogue
      20: "epi: staging block free", 21: "epi: residual in hand", 22: "epi: outputs computed",
      23: "epi: output stores issued", 24: "epi: staging block handed over"}
for c, role, ev in ev_all[:n_ev]:
    if role == 0:
        label = pn.get(ev, str(ev))
    elif role == 1:
        label = f"slot free -> load B block {ev - 10}"
    elif role in MMA:
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
rows = []
for r in MMA:
    if per_role[r]:
        rows += [
            (names[r], "wait on a full slot", spans(r, 4, 5)),
            (names[r], "issue (slot full -> next wait)", spans(r, 5, 4) + spans(r, 5, 2)),
            (names[r], "epilogue (main loop done -> next tile)", spans(r, 2, 1)),
        ]
rows += [
    ("producer", "wait on staged rows", spans(0, 1, 2)),
    ("producer", "gather", spans(0, 2, 6)),
    ("producer", "empty-slot wait + stores", spans(0, 6, 7)),
    ("producer", "end barrier", spans(0, 7, 8)),
    ("loader", "wait on a free stage", spans(4, 2, 1)),
]
print(f"\nlogged window: {window} cycles (CTA 0; each role's log holds at most 512 events)")
for role, what, cyc in rows:
    print(f"{role:9s} {what:40s} {cyc:10d} cycles  {100.0 * cyc / window:5.1f} %")


def tile_intervals(role):
    """Per tile of the warpgroup's log: {event: clock} from its tile start to the next one (complete tiles only)."""
    out, cur = [], None
    for c, _, ev in per_role[role]:
        if ev in (4, 5):
            continue
        if ev == 1:
            if cur is not None:
                cur["next"] = c
                out.append(cur)
            cur = {1: c}
        elif cur is not None:
            cur[ev] = c
    return out


# Per-tile split of each MMA warpgroup's time over the tiles whose main loop and epilogue are both in the log: the wait
# for the other warpgroup's main loop (64 x 128 configuration), the main loop (-> main loop done), then every epilogue
# step (named after the event that ends it), up to the next tile start.
main_iv, epi_iv = {}, {}
for r in MMA:
    tl = tile_intervals(r)
    if not tl:
        continue
    steps = {}
    for t in tl:
        evs = sorted((c, ev) for ev, c in t.items() if ev != "next")
        prev = t[1]
        for c, ev in evs[1:]:
            k = "wait for turn" if ev == 3 else "main loop" if ev == 2 else mn.get(ev, str(ev))
            steps[k] = steps.get(k, 0) + c - prev
            prev = c
        steps["next tile start"] = steps.get("next tile start", 0) + t["next"] - prev
    print(f"\nper tile, {names[r]} warp 0, mean over {len(tl)} tiles (cycles)")
    for k, v in steps.items():
        print(f"  {k:32s} {v / len(tl):9.0f}")
    epi = sum(v for k, v in steps.items() if k not in ("main loop", "wait for turn"))
    print(f"  {'epilogue total (to next start)':32s} {epi / len(tl):9.0f}")
    main_iv[r] = [(t.get(3, t[1]), t[2]) for t in tl if 2 in t]
    epi_iv[r] = [(t[2], t.get(24, t["next"])) for t in tl if 2 in t]
if len(main_iv) == 2:
    # how much of each warpgroup's epilogue (main loop done -> staging handed over) ran while the other warpgroup's
    # main loop did
    for r, o in ((3, 5), (5, 3)):
        tot = sum(b - a for a, b in epi_iv[r])
        ov = sum(max(0, min(b, d) - max(a, c)) for a, b in epi_iv[r] for c, d in main_iv[o])
        if tot:
            print(f"{names[r]} epilogue under {names[o]}'s main loop: {ov} of {tot} cycles ({100.0 * ov / tot:.0f} %)")
