import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from n2nmn_b200 import synth, weights as wts, _lib
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.executor import LayoutExecutor
N,H,Wd,D,T,C=64,10,15,512,12,28
W=wts.init_weights('clevr',H,Wd,D,C,seed=16,bias_std=0.1)
asm=Assembler(synth.vocab_file('clevr'))
for lay in (['_Find','_Exist'], ['_Find','_Find','_EqualNum'], ['_Find','_Describe'], ['_Find','_Transform','_Count']):
    items=[]
    for i in range(8):
        f,w=synth.make_inputs(N,H,Wd,D,T,seed=400+i)
        items.append((torch.from_numpy(f).cuda(),torch.from_numpy(w).cuda(),synth.tokens_from_layouts(asm,[lay]*N,T)))
    ex=LayoutExecutor('clevr',items[0][0],items[0][1],C,asm,weights=W,max_batch=N,max_T=T,max_group=8)
    ex.set_tree_cluster(1)
    single=[ex.forward_device(f,w,t)[0].cpu().numpy().copy() for f,w,t in items]
    for G in (2,4,8):
        outs,_=ex.forward_group([x[0] for x in items[:G]],[x[1] for x in items[:G]],[x[2] for x in items[:G]])
        torch.cuda.synchronize()
        bad=[]
        for g in range(G):
            d=np.abs(outs[g].cpu().numpy()-single[g]).max(axis=1)
            bad += [g*N+q for q in np.nonzero(d>0)[0]]
        print(lay,'G',G,'bad questions',len(bad), bad[:5], bad[-3:])
    del ex
