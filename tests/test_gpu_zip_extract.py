"""zb_zip_extract on crafted archives (zip_extract_inputs): every entry held to the per-entry model on every decoder path, from
host and device sources into host and device slots, alone and beside any other entries.

Which rows of the path table (zb_inflate.cu, Engine::zip_extract) each archive's entries reach, by the launch count of the entry
extracted alone -- intact / overlong (data or stored payload past usize) / cut (input ends early) / crc32 (directory crc32 wrong):

| path                                     | launches alone       | intact                  | overlong          | cut                  | crc32       |
|------------------------------------------|----------------------|-------------------------|-------------------|----------------------|-------------|
| group, stored (k_zip_stored)             | 3                    | s_ok_*, s_ok_after      | s_long            | s_short              | s_crc       |
| group, deflated (k_zip_members)          | 3                    | d_ok_*, w_*             | d_usize_m1, _m258 | d_cut_1..8, _block_end | d_crc     |
| stored big (copy + crc32)                | 2                    | S_ok_w, S_ok_wp1        | S_long            | S_short              | S_crc       |
| stream (block-parallel)                  | L, declined = no     | D_ok_3m, D_ok_w, _wp1   | --                | --                   | D_crc       |
| declined -> group                        | L + 3, declined      | X_fixed_ok, X_stored_ok | X_fixed_m1, _m258 | X_cut_5              | X_fixed_crc |
| declined, 4 GiB or more -> serial        | L + serial           | zeros (4 GiB + 1000)    |                   |                      |             |

L: the launches of zb_inflate_ex(-15, ZB_INF_CHECK_CRC | ZB_INF_NO_SERIAL) on the entry alone.  The block-parallel decoder
delivers only a whole stream that fits the slot, so an overlong or cut entry of the stream row is always declined: those are
X_fixed_m1 / X_cut_5 / X_lie_below, and the stream row keeps the lies that still decode whole (D_usize_p1, D_junk, D_claims_w)."""
import ctypes
import random
import zlib

import pytest

import zip_extract_inputs as X
import zlib_rs_b200 as Z

pytestmark = pytest.mark.gpu
PAT = 0xA5  # what a device slot holds before the call


@pytest.fixture(scope="module")
def eng():
    return Z.Engine(0)


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


_WANT = {}


def wants(name):
    """The model's Want of every entry of archive `name`, for slots at least usize long."""
    if name not in _WANT:
        arc, ents, offs = X.archive(name)
        _WANT[name] = [X.expect_entry(arc, o, e) for e, o in zip(ents, offs)]
    return _WANT[name]


def slots(ents, which, loose):
    """dst_off for `which`: tight slots (exactly usize) or loose ones (37 bytes more)."""
    off = [0]
    for i in which:
        off.append(off[-1] + ents[i].usize + (37 if loose else 0))
    return off


def run(eng, torch, name, which, src_dev=False, dst_dev=False, loose=False):
    """Extract `which` of archive `name`.  Returns (rc, items, [slot bytes], dst_off)."""
    arc, ents, offs = X.archive(name)
    off = slots(ents, which, loose)
    if src_dev:
        d_arc = torch.frombuffer(bytearray(arc), dtype=torch.uint8).cuda()
        a = eng.zip_open((d_arc.data_ptr(), len(arc)), src_on_device=True)
        src = (d_arc.data_ptr(), len(arc))
    else:
        a = eng.zip_open(arc)
        src = arc
    if dst_dev:
        dst = torch.full((max(off[-1], 1),), PAT, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc, _, items = eng.zip_extract(src, a, which, src_on_device=src_dev, dst=dst.data_ptr(), dst_off=off, dst_on_device=True)
        buf = dst.cpu().numpy().tobytes()
    else:
        host = ctypes.create_string_buffer(max(off[-1], 1))
        ctypes.memset(host, PAT, len(host))
        rc, _, items = eng.zip_extract(src, a, which, src_on_device=src_dev, dst=ctypes.addressof(host), dst_off=off)
        buf = host.raw
    a.close()
    return rc, items, [buf[off[k]:off[k + 1]] for k in range(len(which))], off


def check_entry(e, w, r, slot, dst_dev):
    """One entry's result and slot against the model's Want."""
    tag = (e.name, r.status, r.msg.decode(), r.out_bytes, r.in_bytes, r.check)
    assert (r.status, r.msg.decode()) == (w.status, w.msg), tag
    if w.status == X.Z_OK:
        assert (r.out_bytes, r.in_bytes, r.check) == (e.usize, e.csize, e.crc), tag
        assert slot[:e.usize] == w.data, tag
    elif w.status == X.Z_DATA_ERROR:
        assert r.out_bytes <= e.usize and r.in_bytes <= e.csize, tag
        if w.out_bytes is not None:
            assert (r.out_bytes, r.in_bytes) == (w.out_bytes, w.in_bytes), tag
        assert slot[:r.out_bytes] == w.data[:r.out_bytes], tag
        assert r.check == zlib.crc32(slot[:r.out_bytes]), tag
    else:  # refused: nothing decoded
        assert (r.out_bytes, r.in_bytes, r.check) == (w.out_bytes, 0, 0), tag
    n = r.out_bytes if w.status != X.Z_BUF_ERROR else 0
    if dst_dev:
        # nothing past usize is written; behind the output only zeros of a cleared slot may replace the caller's bytes
        assert slot[min(e.usize, len(slot)):] == bytes([PAT]) * (len(slot) - min(e.usize, len(slot))), tag
        assert set(slot[n:e.usize]) <= {PAT, 0}, tag
    else:
        assert slot[n:] == bytes(len(slot) - n), tag


def summary(items, slot_bytes):
    return [(r.status, r.msg, r.out_bytes, r.in_bytes, r.check, s[:r.out_bytes] if r.status != X.Z_BUF_ERROR else b"")
            for r, s in zip(items, slot_bytes)]


@pytest.mark.parametrize("name", X.NAMES)
def test_model_parity_all_sources_and_destinations(eng, torch, name):
    arc, ents, offs = X.archive(name)
    ws = wants(name)
    which = list(range(len(ents)))
    ref = None
    for src_dev in (False, True):
        for dst_dev in (False, True):
            for loose in (False, True):
                rc, items, sl, _ = run(eng, torch, name, which, src_dev, dst_dev, loose)
                for e, w, r, s in zip(ents, ws, items, sl):
                    check_entry(e, w, r, s, dst_dev)
                first = next((w.status for w in ws if w.status), 0)
                assert rc == first
                got = summary(items, sl)
                if ref is None:
                    ref = got
                assert got == ref, (src_dev, dst_dev, loose)


def path_of(eng, arc, e, o, launches):
    """The path table row an entry alone took, from its launch count."""
    if e.flags & 1 or e.method not in (0, 8):
        assert launches == 0
        return "refused"
    if e.method == 0:
        assert launches == (3 if e.csize < X.WARP_MAX else 2), (e.name, launches)
        return "group_stored" if e.csize < X.WARP_MAX else "stored_big"
    if e.usize < X.WARP_MAX:
        assert launches == 3, (e.name, launches)
        return "group_deflated"
    rc1, _, r1 = eng.inflate(arc[o:o + e.csize], e.usize, window_bits=-15, flags=Z.ZB_INF_CHECK_CRC | Z.ZB_INF_NO_SERIAL)
    if rc1 == Z.ZB_E_DECLINED:
        assert launches == r1.gpu_launches + 3, (e.name, launches, r1.gpu_launches)
        return "declined"
    assert launches == r1.gpu_launches, (e.name, launches, r1.gpu_launches)
    return "stream"


ROWS = {  # entries whose row the table in the docstring names
    "s_long": "group_stored", "s_short": "group_stored", "s_crc": "group_stored", "s_ok_1000": "group_stored",
    "d_usize_m1": "group_deflated", "d_cut_3": "group_deflated", "d_crc": "group_deflated", "d_ok_l6": "group_deflated",
    "S_long": "stored_big", "S_short": "stored_big", "S_crc": "stored_big", "S_ok_w": "stored_big",
    "D_ok_3m": "stream", "D_ok_w": "stream", "D_crc": "stream", "D_junk": "stream", "D_usize_p1": "stream", "D_claims_w": "stream",
    "X_fixed_ok": "declined", "X_stored_ok": "declined", "X_fixed_m1": "declined", "X_cut_5": "declined", "X_fixed_crc": "declined",
    "X_too_far": "declined",
}


@pytest.mark.parametrize("name", X.NAMES)
def test_isolation_and_paths(eng, torch, name):
    # every entry's result and slot are the same alone, in reverse, twice over and in random subsets, as in the whole call
    arc, ents, offs = X.archive(name)
    ws = wants(name)
    n = len(ents)
    rc, items, sl, _ = run(eng, torch, name, list(range(n)))
    whole = summary(items, sl)
    full_slots = sl
    seen = {}
    for i in range(n):
        rc, items, sl, _ = run(eng, torch, name, [i])
        assert summary(items, sl) == [whole[i]] and sl[0] == full_slots[i], ents[i].name
        seen[ents[i].name] = path_of(eng, arc, ents[i], offs[i], items[0].gpu_launches)
    for k, row in ROWS.items():
        if k in seen:
            assert seen[k] == row, (k, seen[k])
    rng = random.Random(n)
    calls = [list(range(n))[::-1]] + [[i, i] for i in range(0, n, 3)] + [rng.sample(range(n), rng.randint(2, n)) for _ in range(4)]
    for which in calls:
        for dev in (False, True):
            rc, items, sl, _ = run(eng, torch, name, which, dev, dev, loose=dev)
            for k, i in enumerate(which):
                check_entry(ents[i], ws[i], items[k], sl[k], dev)
                assert summary([items[k]], [sl[k]]) == [whole[i]], (ents[i].name, which)


def test_read_bounds(eng, torch):
    # the bytes a cut payload lacks sit right behind it: in the gap on a device source, as the next selected entry's payload on a
    # host source.  A decoder that reads past the compressed size would end these OK.
    for name, keys in (("bounds", ("d_cut_", "s_short")), ("declined", ("X_cut_5",))):
        arc, ents, offs = X.archive(name)
        ws = wants(name)
        for src_dev in (False, True):
            rc, items, sl, _ = run(eng, torch, name, list(range(len(ents))), src_dev, False)
            for e, w, r in zip(ents, ws, items):
                if e.name.startswith(keys):
                    assert r.status == X.Z_DATA_ERROR and r.msg.decode() == w.msg == e.want, (e.name, src_dev, r.msg)


def test_forged_size_with_caller_slots(eng, torch):
    arc, offs, ents = X.forged_size_archive()
    a = eng.zip_open(arc)
    assert a.entries[1].uncompressed_size == 1 << 40
    off = [0, ents[0].usize, ents[0].usize + 4096, ents[0].usize + 4096 + ents[2].usize]
    host = ctypes.create_string_buffer(off[-1])
    rc, _, items = eng.zip_extract(arc, a, [0, 1, 2], dst=ctypes.addressof(host), dst_off=off)
    assert rc == Z.Z_BUF_ERROR
    assert (items[1].status, items[1].out_bytes, items[1].in_bytes) == (Z.Z_BUF_ERROR, 1 << 40, 0)
    for k in (0, 2):
        w = X.expect_entry(arc, offs[k], ents[k])
        assert items[k].status == 0 and host.raw[off[k]:off[k + 1]] == w.data
    assert host.raw[off[1]:off[2]] == bytes(4096)
    a.close()


def test_deflated_entry_past_4gib(eng, torch):
    # zeros in one fixed-code block: the block-parallel decoder declines it, and with 4 GiB of output or more the entry takes the
    # serial decoder instead of the group.  Held to the model's crc32 and size on the device.
    arc, offs, ents = X.big_zero_archive()
    e = ents[1]
    rc, _, produced, consumed, crc, _ = X.oracle_inflate(arc[offs[1]:offs[1] + e.csize], X.BIG + 1, keep=False)
    assert (rc, produced, consumed) == (X.Z_STREAM_END, X.BIG, e.csize)
    e.crc = crc  # the directory's crc32 is the model's
    arc, offs = X.craft(ents)
    a = eng.zip_open(arc)
    off = [0, ents[0].usize, ents[0].usize + X.BIG + 64, ents[0].usize + X.BIG + 64 + ents[2].usize]
    dst = torch.full((off[-1],), PAT, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc, _, items = eng.zip_extract(arc, a, [0, 1, 2], dst=dst.data_ptr(), dst_off=off, dst_on_device=True)
    r = items[1]
    assert rc == 0 and (r.status, r.out_bytes, r.in_bytes, r.check) == (0, X.BIG, e.csize, crc), (r.status, r.msg, r.out_bytes)
    assert int(dst[off[1]:off[1] + X.BIG].count_nonzero()) == 0
    assert bool((dst[off[1] + X.BIG:off[2]] == PAT).all())
    assert dst[off[0]:off[1]].cpu().numpy().tobytes() == X.expect_entry(arc, offs[0], ents[0]).data
    a.close()
