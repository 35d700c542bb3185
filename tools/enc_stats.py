import os, sys, ctypes as C, numpy as np
os.environ["B2H264_ENC_STATS"]="1"
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")); sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import h264lib
from openh264_b200.binding import BatchEncoder, lib
W,H=1920,1080
S=int(sys.argv[1]) if len(sys.argv)>1 else 16
clip=h264lib.synth_clip(W,H,6); fsz=W*H*3//2
enc=BatchEncoder(W,H,qp=26,fps=30.0,n_streams=S)
L=lib(0); L.b2h264_debug_enc_stats.argtypes=[C.c_void_p,C.c_int]
st=np.zeros(16,np.uint64)
lists=['A skip test + skip cand. intra check','I intra MB','B inter','C intra in P']   # ready lists of k_encode_mbs (enc_kernels.cu: enc_list)
NQ=len(lists)
names=['-',lists[0],lists[1],'-',lists[2],lists[3],'-','-']   # index = stage id (enc_inter.cuh: MBS_*; 3 is not a stage)
for f in range(6):
    enc.encode([clip[f*fsz:(f+1)*fsz]]*S)
    L.b2h264_debug_enc_stats(st.ctypes.data,1)
    t=enc.timing_us()
    if hasattr(L,'b2h264_debug_batch_stats'):
        bt=np.zeros((NQ+1,3),np.uint64); L.b2h264_debug_batch_stats(bt.ctypes.data,1)
        print('   batches [list: count, avg fill, avg cycles]:', {lists[k]:(int(bt[k][0]), round(float(bt[k][1])/max(1,int(bt[k][0])),1), int(bt[k][2]//max(1,bt[k][0]))) for k in range(NQ) if bt[k][0]}, 'leader wait Gcyc', round(float(bt[NQ][2])/1e9,2), 'polls', int(bt[NQ][0])&0xffffffff, 'failed claims', int(bt[NQ][0])>>32, 'idle polls', int(bt[NQ][1]), 'batch Gcyc', round(float(bt[:NQ,2].sum())/1e9,2))
    if hasattr(L,'b2h264_debug_fill_stats') and f>=4:
        nl=C.c_int(); wp=C.c_int(); fs=np.zeros((8,64,2),np.uint64)
        L.b2h264_debug_fill_stats.argtypes=[C.c_void_p,C.POINTER(C.c_int),C.POINTER(C.c_int),C.c_int]
        L.b2h264_debug_fill_stats(fs.ctypes.data,C.byref(nl),C.byref(wp),1)
        fs=fs.reshape(-1)[:nl.value*(wp.value+1)*2].reshape(nl.value,wp.value+1,2)
        for k in range(nl.value):
            if fs[k,:,0].sum(): print('   fill histogram', lists[k], {n:(int(fs[k,n,0]), int(fs[k,n,1]//max(1,fs[k,n,0]))) for n in range(1,wp.value+1) if fs[k,n,0]})
    if hasattr(L,'b2h264_debug_task_wall'):
        tw=np.zeros((NQ,2),np.uint64); L.b2h264_debug_task_wall.argtypes=[C.c_void_p,C.c_int]; L.b2h264_debug_task_wall(tw.ctypes.data,1)
        print('   task wall (barrier -> end of run_task) avg cycles:', {lists[k]: int(tw[k][0]//max(1,tw[k][1])) for k in range(NQ) if tw[k][1]})
    busy=float(sum(st[0::2])); n=float(sum(st[1::2]))
    print('   avg cyc/MB %.0f  utilisation of 1184 warps @1.9GHz: %.2f'%(busy/n, busy/(1184*t[0]*1900.0)))
    print('frame',f,'kernel us',round(t[0]),'dbk',round(t[1]), {names[i]:(int(st[2*i+1]), int(st[2*i]//max(1,st[2*i+1]))) for i in range(7) if st[2*i+1]})
