import sys, os, numpy as np
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("leg-kilo_b200/python","oracle","tests"): sys.path.insert(0, os.path.join(ROOT,p))
import lko, scenes
from legkilo_b200 import Engine, abi
np.set_printoptions(linewidth=200, precision=6)
cfg, blob, pts = scenes.planar_scene()
x0 = abi.default_states(1); P0 = abi.init_cov(1); Q=abi.process_cov_Q(cfg)
o = lko.Oracle(cfg); o.map_import(blob); o.set_filter(x0,P0,Q,np.zeros(1,abi.CLOCK_DTYPE)); o.set_options(gain_mode=1,iters=1,update_map=False)
ro = o.predict_update_point(0.0, pts, debug=True); xo,Po,_,_ = o.get_filter()
eng = Engine(cfg); eng.map_upload(blob)
d = eng.debug_residuals(x0,P0,pts)
m = ro["ok"].astype(bool)
print("key eq", np.array_equal(d["key"],ro["key"]), "ok eq", np.array_equal(d["ok"],ro["ok"]), m.sum())
print("R relerr", np.abs(d["R"][m]/ro["R"][m]-1).max())
print("hz abserr", np.abs(d["h"][m]*d["z"][m,None]-ro["h"][m]*ro["z"][m,None]).max(), "scale", np.abs(ro["h"][m]*ro["z"][m,None]).max())
print("|h| err", np.abs(np.abs(d["h"][m])-np.abs(ro["h"][m])).max(), " |z| err", np.abs(np.abs(d["z"][m])-np.abs(ro["z"][m])).max())
out = eng.scan_update(x0,P0,Q,np.zeros(1,abi.CLOCK_DTYPE),pts,[0,len(pts)],[0.0])
print("delta gpu", lko.boxminus(out["x"],x0)[:9]); print("delta cpu", lko.boxminus(xo,x0)[:9])
# oracle info-form update from GPU rows
o2 = lko.Oracle(cfg); o2.set_filter(x0,P0,Q,None); o2.update_by_points(d["h"][m], d["z"][m], d["R"][m], gain_mode=1)
x2,P2,_,_ = o2.get_filter(); print("delta cpu(gpu rows)", lko.boxminus(x2,x0)[:9])
print("P err", scenes.cov_err(out["P"][0],Po))
import ctypes as C
from legkilo_b200 import lib, _p
part = np.zeros((8,32)); lib().lk_debug_read.argtypes=[C.c_void_p,C.c_int,C.c_void_p,C.c_size_t]
lib().lk_debug_read(eng.h, 0, _p(part), part.nbytes)
tot = part.sum(0)
hh=d["h"][m]; zz=d["z"][m]; RR=d["R"][m]; w=1/RR
A=(hh*w[:,None]).T@hh; b=(hh*w[:,None]).T@zz
iu=np.triu_indices(6)
print("A err", np.abs(tot[:21]-A[iu]).max()/np.abs(A).max()); print("b gpu", tot[21:27]); print("b cpu", b); print("sumR cnt", tot[26], RR.sum(), tot[27])
