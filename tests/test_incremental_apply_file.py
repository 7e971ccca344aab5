"""CPU-only: IncrementalLoader handing whole packet files to apply_file (persia_core applies them on the device) keeps
the order and counters of the decoding loader."""
import os

import numpy as np
import pytest

from persia_b200 import incremental as INC


def _flush(root, name, packets, done=True):
    d = os.path.join(root, name)
    os.makedirs(d)
    for i, p in enumerate(packets):
        with open(os.path.join(d, f"0_{i}.inc"), "wb") as f:
            f.write(p)
    if done:
        open(os.path.join(d, INC.DONE_FILE), "w").close()


def _packet(n, first=1):
    return INC.encode_packet(np.arange(first, first + n, dtype=np.uint64), 4, np.ones((n, 4), np.float32), 5)


def test_apply_file_sees_the_decoding_loaders_files_in_its_order(tmp_path):
    root = str(tmp_path)
    seen_file, seen_dec = [], []

    def apply_file(path):
        seen_file.append(path)
        signs = INC.decode_packet(open(path, "rb").read())[0]  # raises as a device apply would for a bad packet
        return 1, signs.size

    def apply(signs, dims, entries):
        seen_dec.append(int(signs[0]))
        return 1

    by_file = INC.IncrementalLoader(root, apply_file=apply_file)
    by_dec = INC.IncrementalLoader(root, apply)
    files = [_packet(3, 10), _packet(5, 20)] + [_packet(1, 30 + i) for i in range(10)]
    _flush(root, "inc_b", files[:2])
    _flush(root, "inc_a", files[2:] + [_packet(2)[:-1]])  # 11 files in index order (0_10 after 0_9), the last one bad
    _flush(root, "inc_c", [_packet(4)], done=False)
    assert by_file.poll() == by_dec.poll() == ["inc_a", "inc_b"]
    for ld in (by_file, by_dec):
        assert (ld.entries_applied, ld.entries_dropped, ld.failed_files) == (10 + 3 + 5, 12, 1)
    names = [os.path.relpath(p, root) for p in seen_file]
    assert names == [os.path.join("inc_a", f"0_{i}.inc") for i in range(11)] + \
        [os.path.join("inc_b", f"0_{i}.inc") for i in range(2)]
    assert seen_dec == list(range(30, 40)) + [10, 20]


def test_one_of_apply_and_apply_file(tmp_path):
    with pytest.raises(ValueError):
        INC.IncrementalLoader(str(tmp_path))
    with pytest.raises(ValueError):
        INC.IncrementalLoader(str(tmp_path), lambda *a: 0, apply_file=lambda p: 0)
