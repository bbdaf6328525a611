"""Times the device-resident decode of every BASELINE.json workload shape and checks it bit-for-bit.

usage: python tools/bench_configs.py [out.json]"""
import sys, time, json
sys.path.insert(0, ".")
import numpy as np
import claxon_b200 as cb
from claxon_b200 import synth

ctx = cb.Context(n_streams=8)
rows = []
for name, n in (("c2", 1024), ("c3", 8192), ("c4", 11000), ("c5", 256)):
    t0 = time.time(); b = synth.workload(name, n); tg = time.time() - t0
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    dev = ctx.upload(b.data, descs, out_elems)
    dev.decode(0); dev.sync()
    ms = []
    for i in range(5):
        dev.decode(0); dev.sync(); ms.append(dev.kernel_ms())
    out, res = dev.read()
    ok = bool((res["status"] == 0).all())
    for i in range(0, b.n_frames, max(1, b.n_frames // 257)):
        o = int(descs[i]["out_offset"]); lo, hi = int(b.pcm_offsets[i]), int(b.pcm_offsets[i + 1])
        ok &= bool(np.array_equal(out[o:o + hi - lo], b.pcm[lo:hi]))
    m = float(np.median(ms))
    alg = b.data.size + 4 * b.n_samples
    rows.append({"workload": name, "frames": b.n_frames, "samples": b.n_samples, "in_bytes": int(b.data.size),
                 "kernel_ms": m, "msamples_per_s": b.n_samples / m / 1e3, "alg_GBps": alg / m / 1e6, "bit_exact": ok,
                 "gen_s": round(tg, 1)})
    print(rows[-1], flush=True)
    dev.close()
if len(sys.argv) > 1:
    json.dump(rows, open(sys.argv[1], "w"), indent=1)
