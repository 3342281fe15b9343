"""Where does the end-to-end leg spend its time?  One SF10 Q1 lineitem batch (59 986 052 rows, 6.0 GB of Arrow buffers in
pageable host memory) is imported into HBM under different settings of the host packer; every line is the median of 5 imports.
  python scripts/h2d_probe.py [sf]
"""
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 10.0
    import torch
    from datagen import tpch_gpu
    from sail_b200 import engine
    import bench
    cores = bench.host_cores()
    gpu_node = None
    try:
        import pynvml
        pynvml.nvmlInit()
        bus = pynvml.nvmlDeviceGetPciInfo(pynvml.nvmlDeviceGetHandleByIndex(0)).busId
        bus = bus.decode() if isinstance(bus, bytes) else bus
        gpu_node = int(open(f"/sys/bus/pci/devices/{bus[4:].lower()}/numa_node").read())
    except Exception as e:      # noqa: BLE001
        gpu_node = f"? ({e})"
    nodes = {}
    for d in sorted(os.listdir("/sys/devices/system/node")) if os.path.isdir("/sys/devices/system/node") else []:
        if d.startswith("node"):
            nodes[d] = open(f"/sys/devices/system/node/{d}/cpulist").read().strip()
    print(json.dumps({"host_cores": cores, "affinity": len(os.sched_getaffinity(0)), "gpu_numa_node": gpu_node, "numa": nodes}), flush=True)
    ctx0 = engine.Context(0)
    gen = tpch_gpu.generate_buffers(sf, 0, None, (), bench.Q1_COLS, 0)[1] if False else None
    total_sf, chunks = bench.shard_chunks(sf, sf, 0, 1)
    gen = tpch_gpu.generate_buffers(total_sf, chunks[0][0], chunks[0][1], (), bench.Q1_COLS, 0)[1]
    table = gen.host_table()
    batch = table.to_batches()[0]
    nbytes = sum(b.size for c in table.columns for ch in c.chunks for b in ch.buffers() if b is not None)
    del gen
    ctx0.close() if hasattr(ctx0, "close") else None

    def run(label, env, affinity=None):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        old_aff = os.sched_getaffinity(0)
        if affinity:
            os.sched_setaffinity(0, affinity)
        try:
            ctx = engine.Context(0)
            spec = {"op": "filter", "predicate": {"op": "<", "l": {"col": 6}, "r": {"lit": 0, "type": "Date32"}}, "projection": [0]}
            times = []
            for i in range(7):
                op = engine.GpuExec(spec, [batch.schema], ctx)
                ctx.synchronize()
                t0 = time.perf_counter()
                op.push(batch)
                ctx.synchronize()
                times.append(time.perf_counter() - t0)
                op.finish()
                m = op.metrics()
                op.close()
            t = statistics.median(times[2:])
            print(json.dumps({"case": label, "ms": round(t * 1e3, 2), "arrow_GBps": round(nbytes / t / 1e9, 1), "rows_per_s": round(table.num_rows / t / 1e9, 3),
                              "env": env}), flush=True)
            if hasattr(ctx, "close"):
                ctx.close()
        finally:
            os.sched_setaffinity(0, old_aff)
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v

    try:
        import ctypes
        libc = ctypes.CDLL(None, use_errno=True)
        where = {}
        for ci, c in enumerate(table.columns):
            buf = c.chunks[0].buffers()[1]
            for off in (0, buf.size // 2, buf.size - 1):
                page = ctypes.c_void_p((buf.address + off) & ~4095)
                st = ctypes.c_int(-1)
                rc = libc.syscall(279, 0, ctypes.c_ulong(1), ctypes.byref(page), None, ctypes.byref(st), 0)
                where[f"col{ci}@{off * 100 // max(1, buf.size)}%"] = st.value if rc == 0 else f"errno {ctypes.get_errno()}"
        print(json.dumps({"numa_node_of_source_pages": where}), flush=True)
    except Exception as e:      # noqa: BLE001
        print(json.dumps({"numa_node_of_source_pages": str(e)}), flush=True)
    run("warm-up", {})
    run("default (one pass, 256 Ki-row pieces, packers on the source's NUMA node)", {})
    run("packers NOT bound to the source's NUMA node", {"SAILGPU_PACK_NUMA": "0"})
    run("raw bytes (no packing)", {"SAILGPU_H2D_PACK": "0"})
    for th in (8, 16, 32):
        run(f"threads={th}", {"SAILGPU_PACK_THREADS": str(th)})
    for pr in (32768, 131072, 262144):
        run(f"piece_rows={pr}", {"SAILGPU_PACK_PIECE_ROWS": str(pr)})
    for name, cpus in nodes.items():
        aff = set()
        for part in cpus.split(","):
            a, _, b = part.partition("-")
            aff |= set(range(int(a), int(b or a) + 1))
        aff &= os.sched_getaffinity(0)
        if aff:
            run(f"pinned to {name}", {}, aff)
    # plain copies for scale: pageable and pinned cudaMemcpy of one 960 MB column
    import numpy as np
    col = table.column(0).chunks[0].buffers()[1]
    src = np.frombuffer(col, dtype=np.uint8)
    dst = torch.empty(src.size, dtype=torch.uint8, device="cuda")
    tsrc = torch.from_numpy(src)
    for label, t_in in (("cudaMemcpy pageable", tsrc), ("cudaMemcpy pinned", tsrc.pin_memory())):
        ts = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dst.copy_(t_in, non_blocking=True)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        t = statistics.median(ts[1:])
        print(json.dumps({"case": label, "ms": round(t * 1e3, 2), "GBps": round(src.size / t / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
