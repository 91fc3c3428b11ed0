"""One batch of config-2 frames through FramePipeline.run_device (for profiler captures and launch lists).
usage: prof_one.py [batch] [reps] [fft]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch
from passiveradar_b200 import _lib, synth
from passiveradar_b200.frames import FramePipeline

batch = int(sys.argv[1]) if len(sys.argv) > 1 else 16
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
_lib.set_option("fft", int(sys.argv[3]) if len(sys.argv) > 3 else 1)
n, F, R = 2 ** 20, 256, 300
dev = torch.device("cuda", 0)
fr = [synth.make_frame(n, "P1", i) for i in range(4)]
ref_d = torch.from_numpy(np.stack([fr[i % 4][0] for i in range(batch)])).to(dev)
srv_d = torch.from_numpy(np.stack([fr[i % 4][1] for i in range(batch)])).to(dev)
maps = torch.empty((batch, F, R + 1), dtype=torch.complex64, device=dev)
pipe = FramePipeline(n, R, F, batch=batch, nslots=1)
for _ in range(reps):
    pipe.run_device(ref_d, srv_d, maps)
torch.cuda.synchronize()
print("done", float(maps.abs().max()))
