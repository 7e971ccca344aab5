"""The committed RSQRTPS table (scripts/gen_rsqrt_table.py) and the oracle's table mode (tests/rsqrt_oracle.py).  CPU only.

The fixture and the generated device header hold the same entries; the table mode reproduces the reference's own
Adagrad golden vectors bit for bit on any host; and on an Intel host the table model equals the instruction on every
one of the 2^32 input bit patterns."""
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import rsqrt_oracle as RO
from test_oracle_golden import ADAGRAD_GOLD, ADAGRAD_VW_GOLD, _intel, _run

HEADER = os.path.join(RO.ROOT, "persia_b200", "csrc", "pb_rsqrt_table.cuh")


def test_fixture_matches_header():
    with open(HEADER) as f:
        body = f.read().split("kRsqrtIntel[2048] = {", 1)[1].split("};", 1)[0]
    hdr = np.array([int(x, 16) for x in re.findall(r"0x([0-9a-f]{8})u", body)], np.uint32)
    fix = RO.table_entries()
    assert fix.size == 2048 and hdr.size == 2048
    np.testing.assert_array_equal(hdr, fix)
    # every entry is a 12-bit mantissa in [0.5, 1]: rsqrt of [1, 4)
    assert not np.any(fix & ~np.uint32(0x7ff800) & np.uint32(0x7fffff))
    f = fix.view(np.float32)
    assert np.all((f > 0.5) & (f <= 1.0))


@pytest.mark.parametrize("kind,gold", [(1, ADAGRAD_GOLD), (2, ADAGRAD_VW_GOLD)])
def test_table_mode_reproduces_adagrad_golden(oracle, kind, gold):
    # persia-common/src/optim.rs:362-445 (assert_eq! on every f32), on any host CPU
    with RO.table_mode(oracle):
        e = _run(oracle, kind)
    assert e.tobytes() == np.array(gold, np.float32).tobytes()


def test_table_mode_leaves_the_oracle_as_it_was(oracle):
    oracle.set_rsqrt_exact(True)
    want = _run(oracle, 1)
    oracle.set_rsqrt_exact(False)
    with RO.table_mode(oracle):
        oracle.set_rsqrt_exact(True)  # the exact mode is still there inside the block
        assert _run(oracle, 1).tobytes() == want.tobytes()
    assert oracle._lib is not RO.lib(oracle)


def test_table_model_specials(oracle):
    x = np.array([0x00000000, 0x80000000, 0x00000001, 0x807fffff, 0x7f800000, 0xff800000, 0xbf800000,
                  0x7fc00001, 0x7f800001, 0xff800001, 0x3f800000, 0x40800000, 0x3e800000], np.uint32)
    want = [0x7f800000, 0xff800000, 0x7f800000, 0xff800000, 0x00000000, 0xffc00000, 0xffc00000,
            0x7fc00001, 0x7fc00001, 0xffc00001]
    got = RO.rsqrt_table(oracle, x)
    assert [int(v) for v in got[:10]] == want
    # 1, 4 and 1/4: the entry of mantissa 0, exponent moved by -1 and +1
    t0 = int(RO.table_entries()[0])
    assert [int(v) for v in got[10:]] == [t0, t0 - (1 << 23), t0 + (1 << 23)]


@pytest.mark.skipif(not _intel(), reason="the table is Intel's RSQRTPS; other CPUs approximate differently")
def test_table_model_is_the_instruction_on_every_input(oracle):
    RO.lib(oracle)
    parts = 64
    step = (1 << 32) // parts
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:  # (ctypes releases the GIL)
        bad = sum(ex.map(lambda i: RO.mismatches(oracle, i * step, (i + 1) * step), range(parts)))
    assert bad == 0
    x = np.arange(0, 1 << 20, dtype=np.uint32) * np.uint32(4093)  # the array calls agree too, NaNs by their bits
    np.testing.assert_array_equal(RO.rsqrt_table(oracle, x), RO.rsqrt_intrinsic(oracle, x))
