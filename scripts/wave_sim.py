"""CPU model of the multi-commit wave structure on C4 (design tool; tests/test_wave_model.py checks its sequences against the oracle): replays the exact reference sequence while grouping it
into waves the way ccsim_multi.cuh does — per-tile top-M publication, the bar T, the candidate cap, kill-on-full-cell, waves that go on
across non-binding PTS minimum moves — and reports placements per wave and why waves end, for alternative tile layouts / M / caps.

    python scripts/wave_sim.py [--layout contiguous|interleaved] [--m 16] [--cap 256] [--nodelta] [--waves N] [--relax a,b,c]
                               [--levels L]
    KNUM=8 RMAX=3 CF=1 python scripts/wave_sim.py        # the look-ahead rule ccsim_multi.cuh ships (MULTI_RELAX_K / MULTI_RELAX_R)
The placement sequence goes to $WAVE_SIM_OUT (.npy).

C4 specifics used: hostname anti-affinity makes every node single-use, so a node's score never changes during the run."""
import argparse, importlib, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
synth = importlib.import_module("cluster-capacity_b200.synth")

ap = argparse.ArgumentParser()
ap.add_argument("--layout", default="contiguous")
ap.add_argument("--m", type=int, default=16)
ap.add_argument("--cap", type=int, default=256)
ap.add_argument("--grid", type=int, default=132)
ap.add_argument("--nodelta", action="store_true")
ap.add_argument("--waves", type=int, default=0)
ap.add_argument("--n", type=int, default=100_000)
ap.add_argument("--existing", type=int, default=200_000)
ap.add_argument("--zones", type=int, default=64)
ap.add_argument("--racks", type=int, default=1024)
ap.add_argument("--regions", type=int, default=8)
ap.add_argument("--perdomain", type=int, default=-1, help="publish the best node per open domain of this constraint (0 zone, 1 rack, 2 region) instead of the top-M")
ap.add_argument("--relax", default="0,0,0", help="look-ahead per constraint: nodes whose cell is at most this far over the limit are published as dormant candidates")
ap.add_argument("--levels", type=int, default=4, help="candidates on at most this many score levels below the best key; when they span more, the "
                "bar goes up to the lowest key of the lowest level kept (0: no limit)")
args = ap.parse_args()
R = [int(x) for x in args.relax.split(",")]
ADAPT = os.environ.get("ADAPT") == "1"; KNUM = int(os.environ.get("KNUM", "0")); PRECISE = os.environ.get("PRECISE", "1") == "1"; CF = float(os.environ.get("CF", "1"))
if ADAPT: R = [0, 0, 0]
cool = [0, 0, 0]; pen = [4, 4, 4]; RMAX = int(os.environ.get("RMAX", "2"))

snap, tmpl, ctr = synth.c4(n=args.n, n_existing=args.existing, zones=args.zones, racks=args.racks, regions=args.regions)
t = tmpl[0]
n = snap.n
a_cpu = np.asarray(snap.alloc_cpu, dtype=np.int64); a_mem = np.asarray(snap.alloc_mem, dtype=np.int64)
r_cpu = np.asarray(snap.req_cpu, dtype=np.int64); r_mem = np.asarray(snap.req_mem, dtype=np.int64)
nz_cpu = np.asarray(snap.nz_cpu, dtype=np.int64) if hasattr(snap, "nz_cpu") and snap.nz_cpu is not None else r_cpu
nz_mem = np.asarray(snap.nz_mem, dtype=np.int64) if hasattr(snap, "nz_mem") and snap.nz_mem is not None else r_mem
a_pods = np.asarray(snap.alloc_pods, dtype=np.int64); npods = np.asarray(snap.npods, dtype=np.int64)
topo = [np.asarray(c, dtype=np.int64) for c in snap.topo]
cnt = [np.asarray(ctr[c]._keep, dtype=np.int64).copy() for c in range(3)]
host = np.asarray(ctr[3]._keep, dtype=np.int64).copy()
skew = [1, 2, 4]

# scores (static per node in C4)
def least(req, cap):
    return np.where((cap == 0) | (req > cap), 0, ((cap - req) * 100) // np.maximum(cap, 1))
ls = (least(nz_cpu + t.least_cpu, a_cpu) + least(nz_mem + t.least_mem, a_mem)) // 2
f0 = np.minimum((r_cpu + t.bal_cpu) / a_cpu, 1.0); f1 = np.minimum((r_mem + t.bal_mem) / a_mem, 1.0)
bal = ((1 - np.abs((f0 - f1) / 2)) * 100.0).astype(np.int64)
score = t.w_fit * ls + t.w_balanced * bal
IDXB = 20; MASK = (1 << IDXB) - 1
key = ((score + 1) << IDXB) | (MASK - np.arange(n))
fit0 = (a_cpu - r_cpu >= t.req_cpu) & (a_mem - r_mem >= t.req_mem) & (a_pods - npods >= 1) & (host == 0)

grid = args.grid
chunk = (n + grid - 1) // grid
tile = (np.arange(n) // chunk) if args.layout == "contiguous" else (np.arange(n) % grid)
alive = fit0.copy()
mins = [int(c.min()) for c in cnt]
lim = [skew[c] - 1 + mins[c] for c in range(3)]          # count <= lim  (maxSkew - selfMatch + min)

placed = 0; waves = 0; delta = 1 << IDXB; strict_next = False; empty_waves = 0
ends = {"dry_artificial": 0, "dry_T": 0, "rescan": 0, "cap64": 0, "none": 0}
cand_total = 0; hist_acc = []; resc_by = [0, 0, 0]; raised = 0; clamped = 0
seq = []
while True:
    if KNUM > 0: R = [RMAX if (int((cnt[c] == mins[c]).sum()) <= KNUM and int((cnt[c] > lim[c]).sum()) * CF <= int((cnt[c] <= lim[c]).sum())) else 0 for c in range(3)]
    Rw = [0, 0, 0] if strict_next else R
    feas = alive & (cnt[0][topo[0]] <= lim[0] + Rw[0]) & (cnt[1][topo[1]] <= lim[1] + Rw[1]) & (cnt[2][topo[2]] <= lim[2] + Rw[2])
    lim_scan = list(lim)
    unpub_min = [int(cnt[c][cnt[c] > lim[c] + Rw[c]].min()) if (cnt[c] > lim[c] + Rw[c]).any() else (1 << 60) for c in range(3)]
    idx = np.nonzero(feas)[0]
    if len(idx) == 0:
        break
    waves += 1
    k = key[idx]
    order = np.argsort(-k, kind="stable")
    idx = idx[order]; k = k[order]
    tl = tile[idx]
    if args.perdomain >= 0:
        # publish per tile the best node of every (open) domain of the chosen constraint, at most M of them (best first)
        dom = topo[args.perdomain][idx]
        pair = tl * (1 << 20) + dom
        _, first = np.unique(pair, return_index=True)
        isbest = np.zeros(len(idx), bool); isbest[first] = True
        # rank among per-domain bests within the tile
        o2 = np.argsort(tl[isbest], kind="stable")
        tb = tl[isbest][o2]
        st = np.r_[0, np.nonzero(np.diff(tb))[0] + 1]
        rk = np.arange(len(tb)) - np.repeat(st, np.diff(np.r_[st, len(tb)]))
        rank = np.full(len(idx), 1 << 30); pos = np.nonzero(isbest)[0][o2]; rank[pos] = rk
        pub = rank < args.m
        # unseen bound: the best unpublished node of each tile
        unpub = ~pub
        Tlist = 0
        if unpub.any():
            o3 = np.argsort(tl[unpub], kind="stable"); tu = tl[unpub][o3]; ku = k[unpub][o3]
            st3 = np.r_[0, np.nonzero(np.diff(tu))[0] + 1]
            Tlist = int(ku[st3].max())      # keys sorted desc within the tile (stable): first = best unpublished
            Tlist += 1                      # candidates must be strictly above every unseen node
    else:
        o2 = np.argsort(tl, kind="stable")
        tb = tl[o2]
        st = np.r_[0, np.nonzero(np.diff(tb))[0] + 1]
        sizes = np.diff(np.r_[st, len(tb)])
        rk = np.arange(len(tb)) - np.repeat(st, sizes)
        rank = np.empty(len(idx), np.int64); rank[o2] = rk
        pub = rank < args.m
        more = np.repeat(sizes > args.m, sizes)
        lastk = (rank == args.m - 1)
        sel = np.zeros(len(idx), bool); sel[o2] = more
        Tl = k[lastk & sel]
        Tlist = int(Tl.max()) if len(Tl) else 0
    kbest = int(k[0])
    T = Tlist if args.nodelta else max(Tlist, kbest - delta if kbest > delta else 0)
    T0 = T
    if args.levels > 0 and ((kbest >> IDXB) - (k[pub & (k >= T)] >> IDXB) >= args.levels).any():
        T = ((kbest >> IDXB) - (args.levels - 1)) << IDXB; clamped += 1
    c_idx = idx[pub & (k >= T)]; c_key = k[pub & (k >= T)]
    if len(c_idx) > args.cap:
        raised += 1
        T = int(c_key[args.cap - 1])      # more than --cap candidates: the bar is the key of rank cap-1
        keep = c_key >= T; c_idx = c_idx[keep]; c_key = c_key[keep]
    overflowed = T > T0
    C = len(c_idx); cand_total += C
    live = np.ones(C, bool)
    cz = [topo[c][c_idx] for c in range(3)]
    acc = 0; reason = "none"; ran_dry = False; resc_c = -1
    dorm0 = [int((live & (cnt[c][cz[c]] > lim[c])).sum()) for c in range(3)]; live0 = int((live & (cnt[0][cz[0]] <= lim[0]) & (cnt[1][cz[1]] <= lim[1]) & (cnt[2][cz[2]] <= lim[2])).sum())
    while True:
        okc = live & (cnt[0][cz[0]] <= lim[0]) & (cnt[1][cz[1]] <= lim[1]) & (cnt[2][cz[2]] <= lim[2])
        lv = np.nonzero(okc)[0]
        if len(lv) == 0:
            ran_dry = True; reason = "dry_artificial" if T > Tlist else "dry_T"; break
        j = lv[0]                        # keys sorted descending
        w = c_idx[j]; live[j] = False; alive[w] = False
        seq.append(w); acc += 1; placed += 1
        rescan = False
        for c in range(3):
            d = cz[c][j]
            old = cnt[c][d]; cnt[c][d] = old + 1
            if old == mins[c] and not (cnt[c] == mins[c]).any():
                mn = int(cnt[c].min()); newlim = skew[c] - 1 + mn
                hit = (newlim >= unpub_min[c]) if (PRECISE and Rw[c] > 0) else bool(((cnt[c] > lim[c]) & (cnt[c] <= newlim)).any())
                if hit: rescan = True; resc_by[c] += 1; resc_c = c
                mins[c] = mn; lim[c] = newlim
        if rescan: reason = "rescan"; break
        if acc >= 64: reason = "cap64"; break
    ends[reason] += 1
    if ADAPT:
        bad = acc == 0 or (ran_dry and acc <= 2 and sum(dorm0) > live0)
        for c in range(3):
            if cool[c] > 0: cool[c] -= 1
            if bad and Rw[c] > 0 and dorm0[c] * 2 > live0: R[c] = 0; cool[c] = pen[c]; pen[c] = min(pen[c] * 2, 1024)
            elif Rw[c] > 0 and acc >= 8: pen[c] = max(4, pen[c] // 2)
            elif resc_c == c and cool[c] == 0: R[c] = min(R[c] + 1, RMAX)
    if acc == 0:
        if strict_next: break
        strict_next = True; empty_waves += 1
    else: strict_next = False
    hist_acc.append(acc)
    if ran_dry and T > Tlist: delta = min(delta * 2, 1 << 30)
    elif overflowed: delta = max(delta // 2, 1 << 8)
    elif (not ran_dry) and C > args.cap // 2: delta = max(delta - delta // 8, 1 << 8)
    if args.waves and waves >= args.waves: break

h = np.array(hist_acc)
print("layout=%s M=%d cap=%d nodelta=%s perdomain=%d: placed %d in %d waves = %.2f placements/wave; candidates/wave %.1f; ends %s" % (
    args.layout, args.m, args.cap, args.nodelta, args.perdomain, placed, waves, placed / max(1, waves), cand_total / max(1, waves), ends))
print("waves without a placement (relaxed scan hid the feasible nodes):", empty_waves)
print("more than %d candidates in %d waves; candidates over %d levels, bar raised in %d waves" % (args.cap, raised, args.levels, clamped))
print("final R", R, "pen", pen)
print("rescans by constraint (zone, rack, region):", resc_by)
print("placements/wave percentiles 10/50/90/max:", np.percentile(h, [10, 50, 90]).tolist(), int(h.max()))
np.save(os.environ.get("WAVE_SIM_OUT", "/tmp/wave_sim_seq.npy"), np.array(seq, dtype=np.int64))
