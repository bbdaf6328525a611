"""Which frames of a workload leave the fast path.

  python tools/exp_paths.py <workload> <frames>

Decodes one device-resident batch with the fallbacks switched off (Context(no_generic=True, no_wide=...)) and
counts the verdicts the throughput path left behind: 0 = done, -2 = needs the generic kernel, -3 = needs the
i64 second chance.  Then the full path, for its kernel time and its final verdicts."""
import collections
import sys
sys.path.insert(0, ".")
import numpy as np
import claxon_b200 as cb
from claxon_b200 import synth

wl = sys.argv[1] if len(sys.argv) > 1 else "c4"
frames = int(sys.argv[2]) if len(sys.argv) > 2 else 1100
b = synth.workload(wl, frames)
descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
for label, opts in (("no generic, no wide", dict(no_generic=True, no_wide=True)), ("no generic", dict(no_generic=True)),
                    ("full path", {})):
    ctx = cb.Context(lane_per_frame=True, **opts)
    dev = ctx.upload(b.data, descs, out_elems)
    for _ in range(2):
        dev.decode(0); dev.sync()
    out, res = dev.read()
    print(wl, frames, label, "kernel ms", round(dev.kernel_ms(), 3), "verdicts",
          dict(collections.Counter(res["status"].tolist())), flush=True)
    dev.close(); ctx.close()
print("exact", bool(np.array_equal(out[:b.n_samples], b.pcm)) if out_elems == b.n_samples else "n/a")
