"""Times the reference's AMX INT4 MoE (shimmed build, oracle/_ref/libktamx.so) at DeepSeek-V3 expert shapes on THIS host:
8-of-N resident experts per layer-forward, one token, thread ladder.  Prints one JSON object."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.bindings import AmxRef, f32_to_bf16_bits  # noqa: E402

E, K, H, I = int(os.environ.get("AMX_E", 16)), 8, 7168, 2048
assert AmxRef.available(), AmxRef.why_unavailable()
rng = np.random.default_rng(0)
mk = lambda shape: f32_to_bf16_bits(rng.standard_normal(shape, dtype=np.float32))  # noqa: E731
g, u, d = mk((E, I, H)), mk((E, I, H)), mk((E, H, I))
x = f32_to_bf16_bits((rng.standard_normal((1, H)) / 100).astype(np.float32))
w = rng.random((1, K)).astype(np.float32)
out = np.zeros((1, H), np.uint16)
ncpu = len(os.sched_getaffinity(0))
res = {}
for th in sorted({2, 4, 8, ncpu}):
    if th > ncpu:
        continue
    amx = AmxRef.get(th)
    h = amx.moe_create(E, K, H, I, g, u, d)
    ids = [np.stack([rng.permutation(E)[:K]]).astype(np.int64) for _ in range(32)]
    for i in range(5):
        amx.moe_forward(h, ids[i], w, x, out)
    t0 = time.perf_counter(); n = 0
    while time.perf_counter() - t0 < 4.0:
        amx.moe_forward(h, ids[n % 32], w, x, out); n += 1
    dt = (time.perf_counter() - t0) / n
    res[th] = dt * 1e3
    amx.moe_destroy(h)
best = min(res, key=res.get)
print(json.dumps({"what": "reference AMXInt4_MOE (kt-kernel/operators/amx, shimmed numa/hwloc build), 1 token x 8-of-%d experts, H=7168 I=2048" % E,
                  "host_cpus": ncpu, "ms_per_layer_by_threads": {str(k): round(v, 3) for k, v in res.items()}, "best_threads": best,
                  "tok_s_equiv_58_layers": 1.0 / (58 * res[best] * 1e-3), "weights_GBps": 8 * 3 * I * H * 0.5 / (res[best] * 1e-3) / 1e9}))
