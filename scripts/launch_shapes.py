"""Which kernels does a stream of bench scans launch, and with what shapes?  A torch.profiler trace (CUDA
activities) of 3 synchronous and 40 pipelined bench scans (the graphs are captured by the first pipelined
scan, inside the trace); prints the sorted multiset of (kernel, grid, block, shared memory) as one line per
distinct shape with its count.  The trace's shared memory is the dynamic plus the kernel's static amount.
Two builds that launch the same kernels with the same shapes print the same lines: the pipelined graphs'
quarter-of-the-GPU grids and the synchronous calls' full-GPU grids both show here.  Writes the trace to the
directory given as the first argument (default: the current directory)."""
import collections, json, os, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import voxblox_b200 as vb
from voxblox_b200 import scenes

out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
n_sync, n_async = 3, 40
scans = scenes.generate_parallel(scenes.c3_room_scan, range(n_sync + n_async))
dev = torch.device("cuda", 0)
d_xyz = [torch.from_numpy(s[0]).to(dev) for s in scans]
d_rgba = [torch.from_numpy(s[1]).to(dev) for s in scans]
torch.cuda.synchronize()
layer = vb.Layer(0.05, 16, engine_options=vb.EngineOptions(max_blocks=16384, max_points_per_scan=1 << 19, max_updates_per_pass=1 << 24))
integ = vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(default_truncation_distance=0.2), layer)


def args(i):
    return (scans[i][2], scans[i][3]), d_xyz[i].data_ptr(), d_rgba[i].data_ptr(), int(scans[i][0].shape[0])


with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(n_sync):
        integ.integratePointCloudDevice(*args(i))
    for i in range(n_sync, n_sync + n_async):
        integ.integratePointCloudAsync(*args(i))
    layer.sync()
trace = os.path.join(out_dir, "launch_shapes.pt.trace.json")
prof.export_chrome_trace(trace)
ev = [e for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel"]
shapes = collections.Counter((e["name"], tuple(e["args"].get("grid", ())), tuple(e["args"].get("block", ())), e["args"].get("shared memory")) for e in ev)
for (name, grid, block, smem), k in sorted(shapes.items()):
    print(f"{k:5d}  grid={list(grid)} block={list(block)} smem={smem}  {name}")
print(f"kernels {len(ev)}, distinct shapes {len(shapes)}")
