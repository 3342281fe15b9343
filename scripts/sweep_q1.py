"""Sweeps the pipeline-kernel geometry (tile rows / stages / hot groups) for the Q1 fused kernel
on one GPU and prints the CUDA-event kernel time of each configuration (resident data)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["SAILGPU_TIMING"] = "1"
import bench  # noqa: E402
from sail_b200 import engine  # noqa: E402


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 10.0
    ctx = engine.Context(0)
    table = bench.gen_shard(sf, 0, 1).combine_chunks()
    specs = bench.q1_specs()
    bench.SORT_ON_GPU = False
    dev = engine.to_device(table, ctx)
    n = table.num_rows
    configs = [dict(), dict(SAILGPU_RPT="1", SAILGPU_STAGES="2"), dict(SAILGPU_RPT="4", SAILGPU_STAGES="1")]
    for cfg in configs:
        for k in ("SAILGPU_RPT", "SAILGPU_STAGES", "SAILGPU_HOT", "SAILGPU_MINB"):
            os.environ.pop(k, None)
        os.environ.update(cfg)
        try:
            for _ in range(2):
                bench.run_query(ctx, specs, [dev], table.schema)
            tot = launches = 0
            for _ in range(5):
                _, _, kns, kl, _ = bench.run_query(ctx, specs, [dev], table.schema)
                tot += kns
                launches += kl
            ms = tot / 1e6 / launches
            print(f"{cfg}: kernel {ms:.3f} ms  -> {n * 100 / ms / 1e6:.1f} GB/s  ({n / ms / 1e6:.2f} Grows/s)", flush=True)
        except Exception as e:  # noqa: BLE001
            print(f"{cfg}: FAILED {e}", flush=True)
    del dev
    ctx.synchronize()


if __name__ == "__main__":
    main()
