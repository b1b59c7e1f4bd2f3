import sys, ctypes, tempfile, json
from pathlib import Path
import numpy as np
sys.path.insert(0, str(__import__('pathlib').Path(__file__).resolve().parents[1]))
import boxmot_b200 as bb
from boxmot_b200 import _lib
from boxmot_b200.synthetic import bench_stream
from oracle.streams import unit_embeddings
lib=_lib.require_device()
n=int(sys.argv[1]) if len(sys.argv)>1 else 256
img,dets=bench_stream(n,60)
embs=unit_embeddings(dets,96,seed=5)
trk=bb.MultiStreamTracker("deepocsort",n_streams=1,cap_tracks=1024,cap_dets=n,feat_dim=embs[0].shape[1])
ph=(ctypes.c_longlong*16)()
for f in range(20): trk.update([dets[f]],None,[embs[f]])
lib.boxmot_b200_tracker_phase_clocks(trk.handle,0,ph,1)
for f in range(20,60): trk.update([dets[f]],None,[embs[f]])
lib.boxmot_b200_tracker_phase_clocks(trk.handle,0,ph,1)
print({i:ph[i]/40 for i in range(16)}, trk.last_device_ms())
