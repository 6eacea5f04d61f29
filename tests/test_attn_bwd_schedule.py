"""Schedule-level statement of csrc/attention_bwd.cu (HMMA) and csrc/attention_bwd_wgmma.cu (wgmma), both 64-row CTAs, on CPU: the CTA / warp / tile loops, causal and length masks, lse / delta
staging and the GQA accumulation order of the two backward kernels, restated line by line in numpy (not the wmma fragment
addressing, which mirrors the GPU-validated forward kernel) and checked against torch.autograd over the eager attention of
transformers qwen2/modeling_qwen2.py:161-184.  It pins the ALGORITHM the kernels implement: a wrong tile bound or mask in
the CUDA file would have to be wrong here too.  TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np
import pytest
import torch

def ref(q,k,v,do,cu,nh,nkv,d):
    T=q.shape[0]; dq=np.zeros_like(q); dk=np.zeros_like(k); dv=np.zeros_like(v); o=np.zeros_like(q); lse=np.zeros((T,nh))
    for b in range(len(cu)-1):
        a,e=cu[b],cu[b+1]
        qq=torch.tensor(q[a:e]).view(-1,nh,d).double().requires_grad_(True); kk=torch.tensor(k[a:e]).view(-1,nkv,d).double().requires_grad_(True); vv=torch.tensor(v[a:e]).view(-1,nkv,d).double().requires_grad_(True)
        kr=kk.repeat_interleave(nh//nkv,1); vr=vv.repeat_interleave(nh//nkv,1)
        w=torch.einsum("thd,shd->hts",qq,kr)/math.sqrt(d); n=e-a
        m=torch.arange(n)[None]>torch.arange(n)[:,None]; w=w.masked_fill(m[None],float("-inf"))
        out=torch.einsum("hts,shd->thd",w.softmax(-1),vr).reshape(n,nh*d)
        g=torch.autograd.grad(out,[qq,kk,vv],torch.tensor(do[a:e]).double())
        dq[a:e]=g[0].reshape(n,-1).numpy(); dk[a:e]=g[1].reshape(n,-1).numpy(); dv[a:e]=g[2].reshape(n,-1).numpy()
        o[a:e]=out.detach().numpy(); lse[a:e]=torch.logsumexp(w,-1).T.detach().numpy()
    return dq,dk,dv,o,lse
def emul(q,k,v,do,o,lse,cu,nh,nkv,d,max_seqlen,BIG=64,SMALL=64):
    """BIG = rows owned by a CTA, SMALL = rows of the streamed tile: (64, 64) = attention_bwd.cu (4 warps x 16 rows) and
    attention_bwd_wgmma.cu (one warpgroup, m64 fragments); (128, 64) = 128-row CTAs, which no kernel uses: it checks that the result
    of the schedule does not depend on the CTA height (the causal tile ranges and the GQA order are stated per row, not per CTA)."""
    NW=BIG//16
    scale=1/math.sqrt(d); LOG2E=1.4426950408889634; sl2=scale*LOG2E
    T=q.shape[0]; delta=(o.reshape(T,nh,d)*do.reshape(T,nh,d)).sum(-1)
    Q=q.reshape(T,nh,d); K=k.reshape(T,nkv,d); V=v.reshape(T,nkv,d); DO=do.reshape(T,nh,d)
    dq=np.full((T,nh,d),np.nan); dk=np.full((T,nkv,d),np.nan); dv=np.full((T,nkv,d),np.nan)
    tiles=(max_seqlen+BIG-1)//BIG; B=len(cu)-1
    def tile(arr,seq0,r0,ln,h,rows):   # rows zero-filled beyond len
        out=np.zeros((rows,d)); valid=min(rows,ln-r0)
        if valid>0: out[:valid]=arr[seq0+r0:seq0+r0+valid,h]
        return out
    # ---- dq kernel
    for b in range(B):
      seq0=cu[b]; ln=cu[b+1]-cu[b]
      for head in range(nh):
        kvh=head//(nh//nkv)
        for qt in range(tiles):
          q0=qt*BIG
          if q0>=ln: continue
          n_tiles=(min(q0+BIG,ln)+SMALL-1)//SMALL
          qs=tile(Q,seq0,q0,ln,head,BIG); dos=tile(DO,seq0,q0,ln,head,BIG)
          acc=np.zeros((BIG,d))
          for j in range(n_tiles):
            kv0=j*SMALL; ks=tile(K,seq0,kv0,ln,kvh,SMALL); vs=tile(V,seq0,kv0,ln,kvh,SMALL)
            for warp in range(NW):
              if BIG==64 and not (kv0<=q0+warp*16+15): continue      # the HMMA kernel skips fully masked warp tiles
              rows=slice(warp*16,warp*16+16)
              S=qs[rows]@ks.T; dP=dos[rows]@vs.T
              dS=np.zeros((16,SMALL))
              for r in range(16):
                row_g=q0+warp*16+r; ok=row_g<ln
                l2=lse[seq0+row_g,head]*LOG2E if ok else 0; dl=delta[seq0+row_g,head] if ok else 0
                for col in range(SMALL):
                  if ok and kv0+col<=row_g:
                    p=2.0**(S[r,col]*sl2-l2); dS[r,col]=p*(dP[r,col]-dl)*scale
              acc[rows]+=dS@ks
          for r in range(BIG):
            if q0+r<ln: dq[seq0+q0+r,head]=acc[r]
    # ---- dkv kernel
    G=nh//nkv
    for b in range(B):
      seq0=cu[b]; ln=cu[b+1]-cu[b]
      for kvh in range(nkv):
        for kt0 in range(tiles):
          kv0=kt0*BIG
          if kv0>=ln: continue
          it0=kv0//SMALL; nq=(ln+SMALL-1)//SMALL; nI=nq-it0; n_iter=G*nI
          ks=tile(K,seq0,kv0,ln,kvh,BIG); vs=tile(V,seq0,kv0,ln,kvh,BIG)
          dka=np.zeros((BIG,d)); dva=np.zeros((BIG,d))
          for n in range(n_iter):
            head=kvh*G+n//nI; q0=(it0+n%nI)*SMALL
            qs=tile(Q,seq0,q0,ln,head,SMALL); dos=tile(DO,seq0,q0,ln,head,SMALL)
            lse_s=np.zeros(SMALL); dlt_s=np.zeros(SMALL)
            for x in range(SMALL):
              qi=q0+x
              if qi<ln: lse_s[x]=lse[seq0+qi,head]*LOG2E; dlt_s[x]=delta[seq0+qi,head]
            for warp in range(NW):
              rows=slice(warp*16,warp*16+16)
              St=ks[rows]@qs.T; dPt=vs[rows]@dos.T
              P=np.zeros((16,SMALL))
              for r in range(16):
                kv_g=kv0+warp*16+r; kv_ok=kv_g<ln
                for col in range(SMALL):
                  qi=q0+col
                  if kv_ok and qi<ln and kv_g<=qi: P[r,col]=2.0**(St[r,col]*sl2-lse_s[col])
              dva[rows]+=P@dos
              dSt=P*(dPt-dlt_s[None,:])*scale
              dka[rows]+=dSt@qs
          for r in range(BIG):
            if kv0+r<ln: dk[seq0+kv0+r,kvh]=dka[r]; dv[seq0+kv0+r,kvh]=dva[r]
    return dq.reshape(T,-1),dk.reshape(T,-1),dv.reshape(T,-1)


@pytest.mark.parametrize("lens,nh,nkv,d", [([5, 64, 65], 4, 2, 16), ([130, 17, 1], 4, 2, 16), ([200], 2, 1, 16), ([64, 128], 4, 4, 16)])
@pytest.mark.parametrize("big", [64, 128])
def test_backward_schedule_equals_autograd(lens, nh, nkv, d, big):
    rng = np.random.default_rng(sum(lens))
    T = sum(lens)
    cu = np.concatenate([[0], np.cumsum(lens)])
    q, k, v, do = (rng.standard_normal((T, n * d)) for n in (nh, nkv, nkv, nh))
    rdq, rdk, rdv, o, lse = ref(q, k, v, do, cu, nh, nkv, d)
    dq, dk, dv = emul(q, k, v, do, o, lse, cu, nh, nkv, d, max(lens), BIG=big, SMALL=64)
    for got, want in ((dq, rdq), (dk, rdk), (dv, rdv)):
        assert not np.isnan(got).any()                      # every row of every sequence is written exactly by its owner CTA
        assert np.abs(got - want).max() < 1e-12
