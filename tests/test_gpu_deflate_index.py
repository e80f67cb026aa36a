"""The index of a stream built while deflating it (zb_deflate_index, DESIGN §2l).

For every case the call must return what zb_deflate_ex returns (code, bytes, result; launches and time aside), and its index must
serialize to exactly the bytes of zb_index_build on the stream just written (window_bits 15 / -15 / 31, ZB_INF_MEMBERS for BGZF)
and of the independent access-point oracle (tests/indexmodel/index_oracle.c), with every window equal to the input in front of its
point.  Ranges extracted through the index must equal slices of the input."""
import ctypes
import random
import zlib

import pytest

import index_lib as IL
import zlib_rs_b200 as Z
from corpus import silesia_tar, synthetic_mix, xorshift_bytes

pytestmark = pytest.mark.gpu

ZB_E_PARAM, ZB_E_BUF = -2, -5
NOT_LAST, END_PARTIAL, END_BLOCK = 1, 16, 32
SPANS = [32768, 65536, 1 << 20, 1 << 32]
FIELDS = [f for f, _ in Z.DeflateResult._fields_ if f not in ("gpu_launches", "gpu_ms")]


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def _inputs():
    mix = synthetic_mix(1300000, seed=21)
    run = bytearray(mix[:400000])
    run[65536 - 120:65536 + 600] = b"z" * 720        # one 258-byte match straddles the target 65536 (and 2 x 32768)
    return {"mix": mix, "tar": silesia_tar()[:700000], "random": xorshift_bytes(300000), "empty": b"", "short": mix[:20000],
            "kS": mix[:3 * 65536], "kS-1": mix[:3 * 65536 - 1], "kS+1": mix[:3 * 65536 + 1], "run": bytes(run)}


INPUTS = _inputs()

# (name, level, strategy, window_bits, flags, memLevel, all inputs)
CONFIGS = [("L%d_%s" % (lv, k), lv, 0, wb, 0, 8, True) for lv in range(10) for k, wb in (("zlib", 15), ("gzip", 31), ("raw", -15))]
CONFIGS += [("L%d_strategy%d" % (lv, s), lv, s, 15, 0, 8, False) for lv in (6, 9) for s in (1, 2, 3, 4)]
CONFIGS += [("L%d_memlevel%d" % (lv, m), lv, 0, 15, 0, m, False) for lv in (1, 6, 9) for m in (1, 9)]
CONFIGS += [("L%d_wbits%d" % (lv, wb), lv, 0, wb, 0, 8, False) for lv in (1, 6) for wb in (9, 12)]
CONFIGS += [("L3_wbits-12_crc", 3, 0, -12, Z.ZB_FLAG_CHECK_CRC, 8, False)]
CONFIGS += [("L%d_low_parallel_adler" % lv, lv, 0, -15, Z.ZB_FLAG_LOW_PARALLEL | Z.ZB_FLAG_CHECK_ADLER, 8, False) for lv in (1, 2)]
CONFIGS += [("L%d_bgzf" % lv, lv, 0, 31, Z.ZB_FLAG_BGZF, 8, True) for lv in (0, 1, 6, 9)]


def build_params(wb, flags):
    """window_bits and flags of the zb_index_build call that indexes the same stream."""
    if flags & Z.ZB_FLAG_BGZF:
        return 31, Z.ZB_INF_MEMBERS
    return (-15 if wb < 0 else 15 if wb <= 15 else 31), 0


def check_of(data, W):
    return 1 if W < 0 else zlib.adler32(data) if W == 15 else zlib.crc32(data)


def deflate_index_raw(eng, data, level, strategy, wb, flags, span, cap=None):
    """zb_deflate_index through ctypes: (rc, bytes, result, index handle or None)."""
    res = Z.DeflateResult()
    cap = cap if cap is not None else (Z.lib().zb_bgzf_bound(len(data)) if flags & Z.ZB_FLAG_BGZF else Z.lib().zb_deflate_bound(len(data))) + 64
    src = ctypes.create_string_buffer(bytes(data), max(len(data), 1))
    dst = ctypes.create_string_buffer(max(cap, 1))
    h = ctypes.c_void_p(1234)
    rc = Z.lib().zb_deflate_index(eng.h, src, len(data), 0, dst, cap, 0, level, strategy, wb, flags, span, ctypes.byref(res),
                                  ctypes.byref(h))
    return rc, dst.raw[:res.out_bytes], res, h.value


def deflate_ex_raw(eng, data, level, strategy, wb, flags, cap):
    res = Z.DeflateResult()
    src = ctypes.create_string_buffer(bytes(data), max(len(data), 1))
    dst = ctypes.create_string_buffer(max(cap, 1))
    rc = Z.lib().zb_deflate_ex(eng.h, src, len(data), 0, dst, cap, 0, level, strategy, wb, flags, ctypes.byref(res))
    return rc, dst.raw[:res.out_bytes], res


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_index_equals_build_and_oracle(eng, cfg):
    name, level, strategy, wb, flags, ml, every_input = cfg
    W, F = build_params(wb, flags)
    for iname, data in INPUTS.items():
        if not every_input and iname in ("tar", "kS-1", "kS+1"):
            continue
        ref, rres = eng.deflate(data, level=level, strategy=strategy, window_bits=wb, flags=flags, mem_level=ml)
        for span in SPANS:
            out, res, idx = eng.deflate_indexed(data, span=span, level=level, strategy=strategy, window_bits=wb, flags=flags,
                                                mem_level=ml)
            assert out == ref, (name, iname, span)
            for f in FIELDS:
                assert getattr(res, f) == getattr(rres, f), (name, iname, span, f)
            blob = idx.to_bytes()
            rc, dec, ires, bidx = eng.build_index(out, len(data) + 64, span=span, window_bits=W, flags=F)
            assert rc == 0 and dec == data
            assert blob == bidx.to_bytes(), (name, iname, span)
            P, M, odec = IL.oracle_points(out, W, span, bool(F))
            assert odec == data
            assert blob == IL.blob(P, M, data, span, len(out), check_of(data, W), W), (name, iname, span)
            pts = idx.points
            for p in pts:
                assert p["window"] == data[p["out_off"] - p["window_len"]:p["out_off"]], (name, iname, span, p)
            # k_deflate_points, and k_index_windows unless every window is empty
            d = res.gpu_launches - rres.gpu_launches
            assert d == (2 if any(p["window_len"] for p in pts) else 1), (name, iname, span, d)


@pytest.mark.parametrize("kind", ["zlib6", "gzip1", "bgzf6", "bgzf1_random"])
def test_extract_through_the_index(eng, kind):
    data = INPUTS["mix"] if kind != "bgzf1_random" else xorshift_bytes(400000, seed=3)
    level = int(kind[4] if kind.startswith(("zlib", "gzip", "bgzf")) else 6)
    wb = 15 if kind.startswith("zlib") else 31
    flags = Z.ZB_FLAG_BGZF if kind.startswith("bgzf") else 0
    out, res, idx = eng.deflate_indexed(data, span=65536, level=level, window_bits=wb, flags=flags)
    rng = random.Random(len(kind))
    n = len(data)
    ranges = [(rng.randrange(n), rng.choice([1, 100, 4096, 70000, 200000])) for _ in range(3000)]
    ranges += [(k * 65280 - 50, 100) for k in range(1, n // 65280 + 1)]    # across BGZF members
    ranges += [(n - 10, 100), (n, 5), (0, n)]
    want = [data[a:a + ln] for a, ln in ranges]
    for index in (idx, Z.Index.from_bytes(idx.to_bytes())):
        rc, outs, items = eng.extract(out, index, ranges)
        assert rc == 0 and outs == want
        ds = eng.alloc(len(out))
        try:
            eng.to_device(ds, out)
            rc, outs, items = eng.extract(ds, index, ranges, n=len(out), src_on_device=True)
            assert rc == 0 and outs == want
        finally:
            eng.free(ds)


@pytest.mark.parametrize("flags,wb", [(NOT_LAST, -15), (NOT_LAST | END_PARTIAL, -15), (NOT_LAST | END_BLOCK, -15),
                                      (3 << 12 | 5 << 16, -15)])
def test_segments_are_refused(eng, flags, wb):
    rc, out, res, h = deflate_index_raw(eng, INPUTS["short"], 6, 0, wb, flags, 65536)
    assert rc == ZB_E_PARAM and h is None
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_indexed(INPUTS["short"], span=65536, window_bits=wb, flags=flags)
    assert e.value.code == ZB_E_PARAM


@pytest.mark.parametrize("span", [0, 32767, (1 << 32) + 1])
def test_spans_are_refused(eng, span):
    rc, out, res, h = deflate_index_raw(eng, INPUTS["short"], 6, 0, 15, 0, span)
    assert rc == ZB_E_PARAM and h is None


@pytest.mark.parametrize("level,flags", [(1, 0), (6, 0), (0, 0), (6, Z.ZB_FLAG_BGZF)])
def test_small_dst_cap_is_what_deflate_ex_gives(eng, level, flags):
    data = INPUTS["tar"]
    wb = 31 if flags else 15
    ref, rres = eng.deflate(data, level=level, window_bits=wb, flags=flags)
    for cap in (10, len(ref) - 1):
        rc, out, res, h = deflate_index_raw(eng, data, level, 0, wb, flags, 65536, cap=cap)
        rc2, out2, res2 = deflate_ex_raw(eng, data, level, 0, wb, flags, cap)
        assert rc == rc2 == ZB_E_BUF and h is None
        assert res.out_bytes == res2.out_bytes == len(ref)
        small = ctypes.create_string_buffer(cap)
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_indexed(data, span=65536, level=level, window_bits=wb, flags=flags, dst=ctypes.addressof(small), dst_cap=cap)
        assert e.value.code == ZB_E_BUF and e.value.needed == len(ref)
    rc, out, res, h = deflate_index_raw(eng, data, level, 0, wb, flags, 65536, cap=len(ref))
    assert rc == 0 and out == ref and h
    Z.lib().zb_index_free(h)
