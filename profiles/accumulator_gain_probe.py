"""Measures whether the tensor-core accumulation error of the 3xTF32 kernels is a systematic GAIN (the tensor core's fp32
accumulation truncates; the engine adds every 32-wide K block into a round-to-nearest fp32 sum to bound it) or noise: for each
kernel, total relative error vs fp64, the fitted gain <y,ref>/<ref,ref>-1 and the residual once the gain is removed.
    python profiles/accumulator_gain_probe.py"""
import sys, os, torch
sys.path.insert(0, os.getcwd())
from brainmagick_b200 import _lib
from brainmagick_b200._lib import call, ptr, stream
dev="cuda"
def raw(w):
    Cout,Cin,Kw=w.shape
    f=torch.empty(Kw,Cout,Cin,device=dev); g=torch.empty(Kw,Cin,Cout,device=dev)
    call("bm_tc_weight_split", ptr(w), Cout, Cin, Kw, ptr(f), None, ptr(g), None, stream()); return f,g
def probe(name, y, ref):
    y=y.double().flatten(); ref=ref.double().flatten()
    gain=(y@ref)/(ref@ref)-1
    res=((y-(1+gain)*ref).norm()/ref.norm()).item()
    tot=((y-ref).norm()/ref.norm()).item()
    print(f"[{name}] total rel err {tot:.2e}  gain {gain.item():+.2e}  residual after gain {res:.2e}")
torch.manual_seed(0)
status=torch.zeros(1,dtype=torch.int32,device=dev)
for (B,T,Cin,Cout,Kw,label) in [(8,360,320,320,3,"K3 fwd n_adds=360"),(8,360,640,320,3,"K=1920 n_adds=720"),(8,360,320,640,1,"1x1 K=320 n_adds=120"),(8,360,1024,640,1,"1x1 K=1024 n_adds=384")]:
    for dist in ("randn","gelu-like"):
        x=torch.randn(B,T,Cin,device=dev)
        if dist=="gelu-like": x=torch.nn.functional.gelu(x)+x.abs()*0.3
        w=torch.randn(Cout,Cin,Kw,device=dev)/(Cin*Kw)**0.5
        f,_=raw(w)
        y=torch.empty(B,T,Cout,device=dev)
        call("bm_tc_conv1d_persistent", ptr(x), ptr(f), None, 0, B,T,Cin,Cout,Kw,1,1,0,0,0, ptr(y),None,None,None,ptr(status),stream())
        torch.cuda.synchronize()
        ref=torch.nn.functional.conv1d(x.double().permute(0,2,1), w.double(), None, padding=Kw//2).permute(0,2,1)
        probe(label+" "+dist, y, ref)
# the same conv through the fp16-piece entry point
lib=_lib.load()
def f16_ops(x, f):
    amax=torch.empty(2,device=dev)
    call("bm_amax", ptr(x), x.numel(), ptr(amax[0:1]), stream()); call("bm_amax", ptr(f), f.numel(), ptr(amax[1:2]), stream())
    hi=torch.empty(f.shape,device=dev,dtype=torch.float16); lo=torch.empty(f.shape,device=dev,dtype=torch.float16)
    call("bm_f16_split", ptr(f), f.numel(), ptr(amax[1:2]), ptr(hi), ptr(lo), stream()); return amax,hi,lo
for tag in ("fp16-piece weights",):
    for (B,T,Cin,Cout,Kw,label) in [(8,360,320,320,3,"f16 K=960 n_adds=180"),(8,360,640,320,3,"f16 K=1920 n_adds=360"),(8,360,320,640,1,"f16 1x1 K=320 n_adds=60"),(8,360,1024,640,1,"f16 1x1 K=1024 n_adds=192")]:
        for dist in ("randn","gelu-like"):
            x=torch.randn(B,T,Cin,device=dev)
            if dist=="gelu-like": x=torch.nn.functional.gelu(x)+x.abs()*0.3
            w=torch.randn(Cout,Cin,Kw,device=dev)/(Cin*Kw)**0.5
            f,_=raw(w)
            amax,hi,lo=f16_ops(x,f)
            y=torch.empty(B,T,Cout,device=dev)
            call("bm_tc_conv1d_f16", ptr(x), ptr(amax[0:1]), ptr(hi), ptr(lo), ptr(amax[1:2]), None, 0, B,T,Cin,Cout,Kw,1,1,0,0,0, ptr(y),None,None,None,None,ptr(status),stream())
            torch.cuda.synchronize()
            ref=torch.nn.functional.conv1d(x.double().permute(0,2,1), w.double(), None, padding=Kw//2).permute(0,2,1)
            probe(tag+" "+label+" "+dist, y, ref)
# wgrad pair
B,T,M,N,Kw=64,360,320,320,3
dy=torch.randn(B,T,M,device=dev); x=torch.randn(B,T,N,device=dev)
ws=torch.empty(int(_lib.load().bm_tc_wgrad_conv_workspace(B,T,M,N,Kw)),device=dev); dw=torch.empty(M,N,Kw,device=dev)
call("bm_tc_wgrad_conv", ptr(dy),ptr(x),B,T,M,N,N,Kw,1,ptr(ws),ptr(dw),ptr(status),stream()); torch.cuda.synchronize()
ref=torch.zeros(M,N,Kw,dtype=torch.float64,device=dev)
for j in range(Kw):
    s=j-1; lo,hi=max(0,-s),min(T,T-s)
    ref[:,:,j]=torch.einsum("btm,btn->mn", dy.double()[:,lo:hi], x.double()[:,lo+s:hi+s])
chunks=B*T//32; print("wgrad chunks per slice ~", chunks/18)
probe("wgrad pair B=64 (per-slice adds ~ %d)"%(chunks/18*12), dw, ref)
print("status", int(status.item()))
