"""Where a unit's WALL time goes inside k_inflate_fast: bench.py's config-2 batch through an FP_PROF build
(scripts/build_variant.sh prof -DFP_PROF; B200Z_LIB=archive_b200/variants/libb200z_prof.so) -- thread 0's clocks per phase,
and inside the LZ77 pass: each warp's clocks probing against copying, copy turns, ready bytes per turn, looks."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import bench  # noqa: E402

NAMES = ["store wait / loop top", "input wait", "header (thread 0)", "tables", "pass A", "pass A2", "chain walk",
         "false-start count + scan", "pass C", "end of blocks + next fetch", "LZ77", "store issue"]


def main():
    from archive_b200 import _ffi, synth
    L = _ffi.ensure_init(0)
    L.b200z_debug_fast_prof.argtypes = [C.POINTER(C.c_ulonglong)]
    dev = torch.device("cuda", 0)
    n, unit = bench.N_UNITS, bench.UNIT
    w = synth.gzip_workload(n, unit, stream0=int(os.environ.get("B200Z_BENCH_STREAM0", 0)), cache_dir=bench.CACHE)
    blob, moff = w["blob"], w["member_off"]
    in_off = (moff[:-1] + 18).astype(np.uint64)
    in_len = (moff[1:] - moff[:-1] - 18).astype(np.uint32)
    out_off = (np.arange(n, dtype=np.uint64) * np.uint64(unit))
    t = lambda a, dt: torch.from_numpy(a.view(dt)).to(dev)
    d_in = torch.empty(len(blob) + 64, dtype=torch.uint8, device=dev)
    d_in[:len(blob)].copy_(torch.from_numpy(blob.copy()))
    d_out = torch.empty(n * unit, dtype=torch.uint8, device=dev)
    d_io, d_il, d_oo = t(in_off, np.int64), t(in_len, np.int32), t(out_off, np.int64)
    d_oc = torch.full((n,), unit, dtype=torch.int32, device=dev)
    d_ol, d_st, d_us = (torch.zeros(n, dtype=torch.int32, device=dev) for _ in range(3))
    ws_bytes = L.b200z_inflate_workspace_bytes(n, len(blob), n * unit)
    d_ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)

    def step():
        rc = L.b200z_inflate_batch_device(d_in.data_ptr(), d_io.data_ptr(), d_il.data_ptr(), d_out.data_ptr(), d_oo.data_ptr(),
                                          d_oc.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), d_us.data_ptr(), n, d_ws.data_ptr(),
                                          ws_bytes, 0)
        assert rc == 0, _ffi.last_error()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    buf = (C.c_ulonglong * 24)()
    L.b200z_debug_fast_prof(buf)
    reps = 5
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        step()
    e1.record()
    torch.cuda.synchronize()
    L.b200z_debug_fast_prof(buf)
    k = n * reps
    tot = sum(buf[:12])
    print(f"{os.environ.get('B200Z_LIB')}: {e0.elapsed_time(e1) / reps:.2f} ms per pass; clocks per unit {tot / k:.0f}")
    for i, name in enumerate(NAMES):
        print(f"  {name:28s} {buf[i] / k:9.0f}  {100.0 * buf[i] / tot:5.1f} %")
    print("  waited at the closing barrier, mean over the 8 warps (clocks per unit; share of the phase):")
    for j, (name, ph) in enumerate([("pass A", 4), ("pass A2", 5), ("false-start count + scan", 7), ("pass C", 8), ("LZ77", 10)]):
        print(f"  {name:28s} {buf[12 + j] / k / 8:9.0f}  {100.0 * buf[12 + j] / 8 / max(buf[ph], 1):5.1f} %")
    probe, copy, turns, tsum, tmax, looks, fails = buf[17:24]
    print("  LZ77 pass, lane 0 of each warp, mean over the 8 warps (clocks per unit; share of the pass's clocks):")
    print(f"  {'probing':28s} {probe / k / 8:9.0f}  {100.0 * probe / max(probe + copy, 1):5.1f} %")
    print(f"  {'copy turns':28s} {copy / k / 8:9.0f}  {100.0 * copy / max(probe + copy, 1):5.1f} %")
    print(f"  copy turns per unit {turns / k:.0f}; ready bytes per turn: sum {tsum / max(turns, 1):.1f}, longest match "
          f"{tmax / max(turns, 1):.1f}; looks per unit {looks / k:.0f}, failed {100.0 * fails / max(looks, 1):.1f} %")


if __name__ == "__main__":
    main()
