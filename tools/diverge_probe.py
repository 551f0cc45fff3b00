import sys,time,os; sys.path.insert(0,os.getcwd())
import numpy as np
import gorse_b200 as gb
from gorse_b200 import synth
small = len(sys.argv)>1 and sys.argv[1]=="small"
U,I,R,d=(100_000,10_000,1_000_000,64) if small else (1_000_000,100_000,10_000_000,64)
off,items=synth.make_feedback(U,I,R,seed=1000,zipf_s=1.0,exact=True)
rng=np.random.default_rng(1)
P0=(rng.standard_normal((U,d))*0.001).astype(np.float32); Q0=(rng.standard_normal((I,d))*0.001).astype(np.float32)
with gb.Context(0) as ctx, gb.CFModel(ctx,U,I,d,off,items) as m:
    m.set_factors(P0,Q0)
    for ep in range(100):
        m.bpr_epoch(0.05,0.01,R,3000+ep,gb.SCATTER_ATOMIC)
        if ep%10==9:
            P,Q=m.get_factors()
            fin=np.isfinite(Q).all() and np.isfinite(P).all()
            print("small" if small else "c2",ep+1,"finite",fin,"max|Q|",np.sqrt((Q*Q).sum(1)).max() if fin else None,"max|P|",np.sqrt((P*P).sum(1)).max() if fin else None, "nan rows Q",int((~np.isfinite(Q)).any(1).sum()), flush=True)
            if not fin: break
