"""GPU box: where does the persistent solver kernel spend its time? Stamps after every grid barrier (s2b_set_solve_trace)."""
import ctypes as C
import sys
import numpy as np
from solver2d_b200 import capi, device, scenes

base = int(sys.argv[1]) if len(sys.argv) > 1 else 447
scene = sys.argv[2] if len(sys.argv) > 2 else "pyramid"
warm = int(sys.argv[3]) if len(sys.argv) > 3 else 12
P = capi.Solver2D(device.LIB_PATH)
dev = device.Device()
if scene == "pyramid":
    sc = scenes.pyramid(P, "TGS_Soft", base_count=base)
elif scene == "field":
    sc = scenes.pyramid_field(P, "TGS_Soft", count=base, base_count=45)  # `base` = number of 1 035-box piles
else:
    sc = scenes.tumbler(P, "TGS_Soft", grid=base)
dw = device.DeviceWorld.attach(dev, sc.world)
L = dev.lib
L.s2b_set_solve_trace.argtypes = [C.c_void_p, C.c_int]
L.s2b_get_solve_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
L.s2b_get_solve_trace.restype = C.c_int
for _ in range(warm):
    sc.step(1 / 60, 4, 2, True)
L.s2b_set_solve_trace(dw.h, 512)
for _ in range(3):
    dw.flush_l2()
    sc.step(1 / 60, 4, 2, True)
out = np.zeros(512, dtype=np.uint64)
n = L.s2b_get_solve_trace(dw.h, out.ctypes.data, 512)
ns = (out[:n] & np.uint64((1 << 48) - 1)).astype(np.int64)
code = (out[:n] >> np.uint64(48)).astype(np.int64)
dt = np.diff(ns)
names = {0: "body", 1: "flat", 2: "group"}
agg = {}
for c, d in zip(code[1:], dt):
    kind = int(c) >> 8
    # an interval ends at a grid barrier and is labelled with the LAST phase before it (region-local phases that ran since
    # the previous barrier are inside the same interval); bit 7: device-wide step (cut colour), bits 7+6: overflow group,
    # bit 6 alone: a neighbour-synchronised colour step (the interval ends at block 0's neighbour wait, not at a grid barrier)
    tag = {0x80: "/cut", 0xC0: "/ovf", 0x40: "/nbr"}.get(kind & 0xC0, "")
    key = (names.get(kind & 0x3F, "?") + tag, int(c) & 0xFF)
    agg.setdefault(key, []).append(int(d))
print("stamps", n, "total us", (ns[-1] - ns[0]) / 1e3)
for key, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
    print(f"{key[0]:9s} op {key[1]:3d}: n={len(v):3d} total {sum(v)/1e3:8.1f} us  mean {np.mean(v)/1e3:6.2f} us  min {min(v)/1e3:6.2f}  max {max(v)/1e3:6.2f}")
print("sequence (us):", [round(float(d) / 1e3, 2) for d in dt[:60]])
c = dw.counters()
print("constraints", c.constraintCount, "colours", c.groupCount, "overflow", c.overflowCount, "regions", c.regionCount, "cut", c.cutCount,
      "cut colours", c.cutGroupCount, "recoloured", c.recolouredCount, "neighbour-synced blocks", c.neighbourSync, "stage ms", dw.stage_ms(), "kernel ms", dev.lib.s2b_last_solve_kernel_ms(dw.h) if hasattr(dev.lib, "s2b_last_solve_kernel_ms") else None)
