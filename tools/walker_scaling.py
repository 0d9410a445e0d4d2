"""How does the LSD region walker scale with the number of frames in flight? (stage times from the handle's CUDA events)"""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np, torch
import __graft_entry__ as g, synth
pkg = g.load_package()
base = synth.batch(640, 480, 64)
for B in [int(a) for a in sys.argv[1:]] or (132, 513, 1026, 2052, 4104):
    frames = np.concatenate([base] * (B // 64 + 1))[:B]
    d = torch.from_numpy(frames).cuda()
    ls = pkg.LineSegment(40, max_width=640, max_height=480, max_batch=B)
    ls.set_profiling(True)
    for _ in range(2):
        ls.extract_batch_device(d.data_ptr(), B, 640, 480, 640, 640 * 480); ls.sync()
    st = ls.stage_ms()
    print(B, {k: round(v, 2) for k, v in st.items()}, "walker us/frame", round(st["lsd_regions"] * 1e3 / B, 1), flush=True)
    del ls, d
    torch.cuda.empty_cache()
