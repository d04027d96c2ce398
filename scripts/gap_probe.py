"""How long do the in-order stages sit idle between scans?  A torch.profiler trace (CUDA activities) of
40 pipelined bench scans; from it, the median gap between one scan's walk (k_rays_emit_warp .. k_assign) and
the next scan's, and between one scan's k_apply and the next one's.  Writes the trace to the directory given
as the first argument (default: the current directory)."""
import json, os, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import voxblox_b200 as vb
from voxblox_b200 import scenes

out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
n_warm, n = 10, 40
scans = scenes.generate_parallel(scenes.c3_room_scan, range(n_warm + n))
dev = torch.device("cuda", 0)
d_xyz = [torch.from_numpy(s[0]).to(dev) for s in scans]
d_rgba = [torch.from_numpy(s[1]).to(dev) for s in scans]
layer = vb.Layer(0.05, 16, engine_options=vb.EngineOptions(max_blocks=16384, max_points_per_scan=1 << 19, max_updates_per_pass=1 << 24))
integ = vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(default_truncation_distance=0.2), layer)


def submit(i):
    integ.integratePointCloudAsync((scans[i][2], scans[i][3]), d_xyz[i].data_ptr(), d_rgba[i].data_ptr(), int(scans[i][0].shape[0]))


for i in range(n_warm):
    submit(i)
layer.sync()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(n_warm, n_warm + n):
        submit(i)
    layer.sync()
trace = os.path.join(out_dir, "gap_probe.pt.trace.json")
prof.export_chrome_trace(trace)
ev = [e for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel"]


def spans(first, last):
    """[start, end] of each scan's run from kernel `first` to kernel `last`, in time order"""
    a = sorted(e["ts"] for e in ev if first in e["name"])
    b = sorted(e["ts"] + e["dur"] for e in ev if last in e["name"])
    return np.array(a[: min(len(a), len(b))]), np.array(b[: min(len(a), len(b))])


res = {"scans": n, "kernels": len(ev)}
for name, first, last in (("walk", "vbx::k_back_begin(", "vbx::k_assign("), ("apply", "vbx::k_apply(", "vbx::k_apply(")):
    s, e = spans(first, last)
    gap = s[1:] - e[:-1]
    res[name] = {"median_busy_us": round(float(np.median(e - s)), 2), "median_gap_us": round(float(np.median(gap)), 2),
                 "p90_gap_us": round(float(np.percentile(gap, 90)), 2), "median_pace_us": round(float(np.median(np.diff(s))), 2)}
print(json.dumps(res))
