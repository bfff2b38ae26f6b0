"""CPU replay of the blend traversals of config 3 with the C oracle (about 25 s on 8 cores): for each 16x16 tile, the
entries a one-warp traversal visits, counting only entries that exact tile culling keeps -- three separate passes (main,
objects-only, background-only) against one main-list pass whose class streams continue past it on their sub-lists
(f_obj_res / f_bg_res: the entries left after the main stream's last one).  Developer tool, next to depth_stats.py."""
import sys, time, numpy as np
sys.path.insert(0, ".")  # run from the repository root
import street_gaussians_ns_b200.synthetic as syn
from oracle import oracle_c
t0 = time.time()
fr = syn.config_frame(3)
orc = oracle_c.Oracle(fr)
fw = orc.forward(class_renders=True)
H, W = fr.camera.height, fr.camera.width
print("forward", fw.N, fw.M, round(time.time() - t0, 1), "s", file=sys.stderr)
xy, con, op = fw.xys, fw.conics, fw.opac
ids, bins = fw.sorted_ids, fw.tile_bins
isobj = (ids < 0) if ids.min() < 0 else None
print("ids min", ids.min(), "fields", [k for k in vars(fw)], file=sys.stderr)
cls = fw.cls.astype(np.int64)
tx_n, ty_n = (W + 15) // 16, (H + 15) // 16
P = H * W
fi = fw.final_idx.reshape(H, W); oi = fw.obj_idx.reshape(H, W); bi = fw.bg_idx.reshape(H, W)
todo = (fw.bg_idx.reshape(H, W) != fi) | (fw.bg_T.reshape(H, W) != fw.final_T.reshape(H, W))
print("cls values", np.unique(cls), "todo px", int(todo.sum()), file=sys.stderr)
yy, xx = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
acc = dict(main=0, obj=0, bg=0, f_main=0, f_obj_res=0, f_bg_res=0, union=0, listed=0)
acc_raw = dict(acc)
for t in range(tx_n * ty_n):
    b, e = int(bins[t, 0]), int(bins[t, 1])
    if e <= b: continue
    ty, tx = divmod(t, tx_n)
    sl = (slice(ty * 16, min(ty * 16 + 16, H)), slice(tx * 16, min(tx * 16 + 16, W)))
    km = int(fi[sl].max()); ko = int(oi[sl].max())
    kb = int(bi[sl][todo[sl]].max()) if todo[sl].any() else -1
    kmax = max(km, ko, kb)
    if kmax < b: continue
    g = ids[b:kmax + 1].astype(np.int64) & 0x7fffffff
    py = (ty * 16 + yy).reshape(-1)[None, :] + 0.5; px = (tx * 16 + xx).reshape(-1)[None, :] + 0.5
    dx = px - xy[g, 0:1]; dy = py - xy[g, 1:2]
    a, bb, c = con[g, 0:1], con[g, 1:2], con[g, 2:3]
    sig = 0.5 * (a * dx * dx + c * dy * dy) + bb * dx * dy
    al = op[g][:, None] * np.exp(-sig)
    kept = ((sig >= 0) & (al >= 1 / 255)).any(axis=1)
    ob = cls[g] == 1
    idx = np.arange(b, kmax + 1)
    def cnt(m, lo, hi):  # kept entries with mask m and index in [lo, hi]
        s = (idx >= lo) & (idx <= hi) & kept & m
        return int(s.sum())
    allm = np.ones_like(ob)
    acc["listed"] += e - b
    acc["main"] += cnt(allm, b, km); acc["obj"] += cnt(ob, b, ko); acc["bg"] += cnt(~ob, b, kb)
    acc["f_main"] += cnt(allm, b, km); acc["f_obj_res"] += cnt(ob, km + 1, ko); acc["f_bg_res"] += cnt(~ob, km + 1, kb)
    acc["union"] += cnt(allm, b, kmax)
print(acc)
print({"today_fwd": acc["main"] + acc["obj"] + acc["bg"], "fused_fwd": acc["f_main"] + acc["f_obj_res"] + acc["f_bg_res"],
       "today_bwd(main+obj)": acc["main"] + acc["obj"], "fused_bwd(main+obj res)": acc["f_main"] + acc["f_obj_res"],
       "secs": round(time.time() - t0, 1)})
