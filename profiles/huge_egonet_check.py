# GPU: spectral parity of the cluster path on explicit huge ego-nets (n = 520, 1500, 3300)
import os, sys, ctypes as C, numpy as np, torch
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT); sys.path.insert(0, os.path.join(_ROOT, 'tests'))
from gcc_b200 import _lib
from gcc_b200.datasets import synthetic
from gcc_b200.datasets.graph_dataset import BatchBuffers
from test_gpu_parity import _fill_batch, _spectral_check
graphs = [synthetic.chung_lu(560, 1500, exponent=0.8, seed=3), synthetic.chung_lu(1700, 5000, exponent=0.9, seed=4),
          synthetic.chung_lu(3500, 9000, exponent=0.9, seed=5), synthetic.star_graph(700)]
subs = [dict(indptr=g.indptr.astype(np.int32), indices=g.indices.astype(np.int32), n=g.num_nodes) for g in graphs]
print([s['n'] for s in subs])
B = 2
N = max(subs[0]['n'] + subs[1]['n'], subs[2]['n'] + subs[3]['n']); E = 2 * max(len(s['indices']) for s in subs) + 8
buf = BatchBuffers(B, N + 8, E + 8 + 20000, 32, 64, 'cuda')
_fill_batch(buf, [subs[:2], subs[2:]])
lib = _lib.get()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for rep in range(2):
    ev[0].record()
    _lib.check(lib.gccb_posenc(C.byref(buf.c), 32, 0, _lib.dptr(buf.pos), _lib.dptr(buf.eigvals), _lib.dptr(buf.ws_posenc), buf.ws_posenc.numel(), _lib.stream_ptr()))
    ev[1].record(); torch.cuda.synchronize(); print('posenc ms', ev[0].elapsed_time(ev[1]))
print('flags', int(buf.flags.item()))
raw = buf.pos.cpu().numpy(); eig = buf.eigvals.cpu().numpy(); noff = buf.node_off.cpu().numpy()
for i, s in enumerate(subs):
    v, gi = divmod(i, 2)
    try:
        _spectral_check(s, raw[v, noff[v, gi]:noff[v, gi + 1]], eig[v * B + gi], tol_l=5e-5); print('ok', s['n'])
    except AssertionError as e:
        print('FAIL', s['n'], str(e)[:150])
