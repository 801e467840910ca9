"""Error of every fp32 tensor-core mode against an fp64 product, on the HOST-EMULATED library (tests/emu): operand
splitting, pass order and the kc-blocked summation are the product's; the accumulator inside a block is a plain fp32
FMA chain, NOT the tensor core's truncating one (that part is what tools/accuracy_probe.py measures on an H100).
  LASER_B200_LIB=tests/emu/_build/liblaser_b200_hostemu.so LASER_B200_EMU=1 python tools/emulated_accuracy.py [M N K]
"""
import sys, numpy as np
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, ROOT)
import laser_b200 as L, oracle as O
from emu_driver import D, rnd
import sys as _s
M,N,K=[int(v) for v in _s.argv[1:4]] if len(_s.argv)>3 else (257,260,520)
for lo,hi in ((0,1),(-.1,.1)):
    a,b=rnd((M,K),1,lo,hi),rnd((K,N),2,lo,hi)
    ex=a.astype(np.float64)@b.astype(np.float64)
    for path in (L.PATH_TF32X3,L.PATH_F16X3):
        c=np.full((M,N),np.nan,np.float32)
        L.gemm_strided(M,N,K,1.0,D(a),K,1,D(b),N,1,0.0,D(c),N,1,path=path)
        e=np.abs(c-ex)
        print(lo,hi,L.PATH_NAMES[path],"normwise %.2e max_rel %.2e mre %.2e"%(np.linalg.norm(c-ex)/np.linalg.norm(ex),(e/np.abs(ex)).max(),(e/np.abs(ex)).mean()))
