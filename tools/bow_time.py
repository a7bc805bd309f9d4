"""CUDA-event time of the batched SearchByBoW (160 pairs, 2000 x 2000, one vocabulary node) — whole call and per kernel under
ncu:  python tools/bow_time.py"""
import ctypes, importlib, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
pkg = importlib.import_module("self_commit_orb-slam2_b200")
F, cap, n = 160, 2048, 2000
m = pkg.ORBmatcher(0.7, True, max_features=cap, max_batch=F)
g = torch.Generator(device="cuda").manual_seed(1)
desc = torch.randint(0, 256, (F + 1, cap, 32), dtype=torch.uint8, device="cuda", generator=g)
node = torch.zeros((F + 1, cap), dtype=torch.int32, device="cuda")
valid = torch.ones((F + 1, cap), dtype=torch.uint8, device="cuda")
ang = torch.rand((F + 1, cap), device="cuda") * 360
cnt = torch.full((F + 1,), n, dtype=torch.int32, device="cuda")
match = torch.zeros((F, cap), dtype=torch.int32, device="cuda")
nm = torch.zeros(F, dtype=torch.int32, device="cuda")
L, vp = pkg.lib(), ctypes.c_void_p
st = torch.cuda.Stream()
def run():
    pkg._check(L.b2s_search_by_bow_device(m._h, F, vp(desc.data_ptr()), vp(node.data_ptr()), vp(valid.data_ptr()), vp(ang.data_ptr()),
                                          vp(cnt.data_ptr()), cap, vp(desc[1:].data_ptr()), vp(node[1:].data_ptr()), None,
                                          vp(ang[1:].data_ptr()), vp(cnt[1:].data_ptr()), cap, 50, 0.7, 0, 1,
                                          vp(match.data_ptr()), vp(nm.data_ptr()), vp(st.cuda_stream)))
for _ in range(3):
    run()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(st)
for _ in range(10):
    run()
e1.record(st)
torch.cuda.synchronize()
print("ms per batched call: %.3f" % (e0.elapsed_time(e1) / 10), "matches", int(nm.sum()))
