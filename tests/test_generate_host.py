"""Host-only logic of generate.py's node export: shard splitting, `--gpu` parsing and `--nodes` files."""
import numpy as np
import pytest

import generate


@pytest.mark.parametrize("n,B,workers", [(1000, 256, 1), (1000, 256, 3), (1024, 256, 4), (1000, 256, 7),
                                         (5, 8, 3), (257, 256, 2), (2560, 256, 3)])
def test_shards_are_contiguous_batch_aligned_and_cover_every_row_once(n, B, workers):
    shards = generate.split_shards(n, B, workers)
    assert len(shards) == workers
    assert shards[0][0] == 0 and shards[-1][1] == n
    for (lo, hi), (lo2, _) in zip(shards, shards[1:]):
        assert hi == lo2                                       # contiguous, in order
    for lo, hi in shards:
        assert lo <= hi and (lo % B == 0 or lo == hi == n)     # a shard starts on a batch boundary, or is empty
        assert hi == n or hi % B == 0                          # only the shard that ends the rows ends short
    covered = np.concatenate([np.arange(lo, hi) for lo, hi in shards])
    assert np.array_equal(covered, np.arange(n))
    sizes = [-(-(hi - lo) // B) for lo, hi in shards]          # batches per shard differ by at most one
    assert max(sizes) - min(sizes) <= 1


def test_more_workers_than_batches_leaves_the_extra_workers_empty():
    shards = generate.split_shards(600, 256, 5)                # 3 batches
    assert shards == [(0, 256), (256, 512), (512, 600), (600, 600), (600, 600)]


def test_gpu_option_takes_one_id_or_a_list():
    assert generate.parse_gpus(None) == [0]
    assert generate.parse_gpus(1) == [1]
    assert generate.parse_gpus([0, 0, 1]) == [0, 0, 1]
    with pytest.raises(ValueError):
        generate.parse_gpus([-1])
    base = ["--load-path", "ckpt.pth"]
    assert generate.parse_args(base).gpu is None
    assert generate.parse_args(base + ["--gpu", "2"]).gpu == [2]
    assert generate.parse_args(base + ["--gpu", "0", "0", "1"]).gpu == [0, 0, 1]
    a = generate.parse_args(base)
    assert a.prefetch == 4 and a.nodes is None and a.batch_size == 256
    assert generate.parse_args(base + ["--prefetch", "0"]).prefetch == 0


def test_nodes_file_text_and_npy(tmp_path):
    ids = np.array([7, 3, 3, 0, 12], dtype=np.int64)
    txt = tmp_path / "ids.txt"
    txt.write_text("7\n3 3\n0\n\n12\n")
    assert np.array_equal(generate.read_nodes(str(txt)), ids)
    npy = tmp_path / "ids.npy"
    np.save(npy, ids.astype(np.int32))
    got = generate.read_nodes(str(npy))
    assert got.dtype == np.int64 and np.array_equal(got, ids)


@pytest.mark.parametrize("content,arr", [("1 2 x\n", None), ("", None), ("1.5\n", None),
                                         (None, np.zeros((2, 2), np.int64)), (None, np.array([0.5, 1.0]))])
def test_nodes_file_rejects_what_is_not_a_list_of_integer_ids(tmp_path, content, arr):
    if arr is None:
        p = tmp_path / "ids.txt"
        p.write_text(content)
    else:
        p = tmp_path / "ids.npy"
        np.save(p, arr)
    with pytest.raises(ValueError):
        generate.read_nodes(str(p))
