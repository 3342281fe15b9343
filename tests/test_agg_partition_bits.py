"""Partitioned mode of the hash aggregate (engine.cu, PipelineOp) sends state rows to key-hash partitions with RepartitionOp's
hash (pipeline.cu partition_of, mirrored by oracle/ops.py hash_partition_ids) and merges every partition in a group table of its
own, whose slot is the low bits of another hash of the same key (pipeline.cu pack_key).  If the two shared bits, the keys of one
partition would all fall into 1/P of their table's slots.  This pins, on the CPU, that they do not: within each partition the
keys spread over every slot residue."""
import numpy as np

from oracle import ops

SEED = np.uint64(0x243F6A8885A308D3)      # pack_key's initial hash


def probe_hash_int64(k: np.ndarray) -> np.ndarray:
    """the group table's hash of one never-null Int64 key (pack_key: h = mix64(seed ^ key word))"""
    return ops.mix64(SEED ^ k.astype(np.uint64))


def partition_hash_int64(k: np.ndarray) -> np.ndarray:
    """RepartitionOp's hash of one Int64 key column (h = mix64(0 ^ mix64(value)))"""
    return ops.mix64(np.zeros(len(k), dtype=np.uint64) ^ ops.mix64(k.astype(np.uint64)))


def test_partition_hash_mirrors_the_oracle():
    import pyarrow as pa
    k = np.arange(-5000, 5000, dtype=np.int64) * 7919
    b = ops.batch_from_arrow(pa.table({"k": pa.array(k)}))
    want = ops.hash_partition_ids(b, [{"col": 0}], 64)
    assert np.array_equal((partition_hash_int64(k) % np.uint64(64)).astype(np.int64), want)


def test_partition_and_probe_use_independent_bits():
    n_parts, slots = 16, 1 << 14
    k = np.arange(1 << 20, dtype=np.int64)            # dense keys: the usual shape of a high-cardinality GROUP BY
    part = (partition_hash_int64(k) % np.uint64(n_parts)).astype(np.int64)
    slot = (probe_hash_int64(k) & np.uint64(slots - 1)).astype(np.int64)
    for p in range(n_parts):
        s = slot[part == p]
        # every residue of the slot modulo P is used about equally (clustering would leave one residue only)
        res = np.bincount(s % n_parts, minlength=n_parts)
        assert res.min() > 0.8 * len(s) / n_parts, (p, res)
        # the keys of one partition reach nearly every slot of a table of their own: 2^16 keys over 2^14 slots
        assert len(np.unique(s)) > 0.95 * slots
