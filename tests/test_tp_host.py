"""The tensor-parallel exchange of include/vptq_b200.h, host-side checks (no GPU needed).

vptq_b200_quant_gemv_multi_tp must refuse an exchange whose slots lie outside its epoch / flag arrays, or whose
stores would be misaligned: the tagged format stores 16-byte words to ys[l] and to every peer_y[l][r]; the plain
format stores 16-byte vectors to peer_y[l][r] + o whenever the local ys[l] + o is aligned.  The addresses here are
fake and every descriptor carries a wrong struct_size, so no version of the library can reach a launch with them:
the exchange checks must come first and name the problem.
"""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _desc(**over):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc) + 8          # wrong on purpose: validate() refuses it
    base = dict(dtype=0, in_features=1024, out_features=512, vector_len=8, num_centroids=65536,
                num_res_centroids=256, num_codebooks=1, group_size=1024, outlier_size=0, outlier_vector_len=-1,
                num_outlier_centroids=-1, indices=0x10000, index_stride_codebook=64 * 768, index_stride_row=768,
                centroids=0x20000, centroid_stride=65536 * 8, res_centroids=0x30000, res_centroid_stride=2048)
    base.update(over)
    for k, v in base.items():
        setattr(d, k, v)
    return d


Y = 0x7000_0000          # local output slice (16-byte aligned)
PEER = 0x9000_0000       # rank r's buffer: PEER + r * 0x10_0000 (+ the same slice offset)


def _exchange(world=4, rank=1, fmt=0, slot=1, wait_slot=0, num_slots=4, n=2, peer_off=0):
    from vptq_b200 import native
    ex = native.TpExchange()
    ex.struct_size = ctypes.sizeof(native.TpExchange)
    ex.world, ex.rank, ex.slot, ex.wait_slot = world, rank, slot, wait_slot
    for l in range(n):
        for r in range(world):
            ex.peer_y[l][r] = PEER + r * 0x10_0000 + l * 0x1000 + peer_off
    for r in range(world):
        ex.peer_flags[r] = 0xA000_0000 + r * 0x1000
    ex.epoch, ex.done, ex.error = 0xB000_0000, 0xB000_1000, 0xB000_2000
    ex.format, ex.num_slots = fmt, num_slots
    return ex


def _call(ex, ys, n=None):
    from vptq_b200 import native
    n = len(ys) if n is None else n
    descs = [_desc() for _ in range(n)]
    darr = (ctypes.POINTER(native.LinearDesc) * n)(*[ctypes.pointer(d) for d in descs])
    yarr = (ctypes.c_void_p * n)(*ys)
    sarr = (ctypes.c_int64 * n)(*[512] * n)
    rc = native.lib().vptq_b200_quant_gemv_multi_tp(n, darr, 0x5000_0000, 1024, yarr, sarr, 1, ctypes.byref(ex),
                                                    0x6000_0000, 1 << 20, 0, None)
    return rc, native.last_error()


YS = [Y, Y + 0x1000]


@pytest.mark.parametrize("fmt", [0, 1])
def test_a_valid_exchange_reaches_the_descriptor_check(fmt):
    """Control: with every exchange rule met, the (deliberately wrong) descriptor is what gets refused."""
    rc, msg = _call(_exchange(fmt=fmt), YS)
    assert rc == -1 and "struct_size" in msg and "ABI mismatch" in msg, msg
    rc, msg = _call(_exchange(fmt=fmt, world=1, rank=0, wait_slot=-1, slot=0, num_slots=1), YS)
    assert rc == -1 and "struct_size" in msg, msg


@pytest.mark.parametrize("off", [2, 4, 8, 14])
def test_tagged_local_y_must_be_16_byte_aligned(off):
    rc, msg = _call(_exchange(fmt=1), [Y, Y + 0x1000 + off])
    assert rc == -1 and "VPTQ_TP_TAGGED needs ys[1] 16-byte aligned" in msg, msg


@pytest.mark.parametrize("off", [2, 8])
@pytest.mark.parametrize("which", ["local", "peer"])
def test_tagged_peer_y_must_be_16_byte_aligned(off, which):
    ex = _exchange(fmt=1)
    r = 1 if which == "local" else 3       # entry [rank] is the local tagged buffer, also written
    ex.peer_y[0][r] += off
    rc, msg = _call(ex, YS)
    assert rc == -1 and f"VPTQ_TP_TAGGED needs peer_y[0][{r}] 16-byte aligned" in msg, msg


@pytest.mark.parametrize("off", [2, 6, 8, 12])
def test_plain_peer_y_must_be_congruent_to_y_modulo_16(off):
    ex = _exchange(fmt=0)
    ex.peer_y[1][2] += off
    rc, msg = _call(ex, YS)
    assert rc == -1 and "peer_y[1][2] - ys[1] must be a multiple of 16 bytes" in msg, msg
    # the same offset on the local slice AND every peer is a legal layout (element-wise stores): accepted
    rc, msg = _call(_exchange(fmt=0, peer_off=off), [Y + off, Y + 0x1000 + off])
    assert rc == -1 and "struct_size" in msg, msg


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("slot,num_slots", [(0, 0), (3, 3), (4, 2), (1, -1)])
def test_slot_must_lie_inside_num_slots(fmt, slot, num_slots):
    rc, msg = _call(_exchange(fmt=fmt, slot=slot, wait_slot=-1, num_slots=num_slots), YS)
    assert rc == -1 and "0 <= slot < num_slots" in msg, msg


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("wait_slot", [4, 5, -2, -100])
def test_wait_slot_must_be_minus_one_or_inside_num_slots(fmt, wait_slot):
    rc, msg = _call(_exchange(fmt=fmt, wait_slot=wait_slot, num_slots=4), YS)
    assert rc == -1 and "-1 <= wait_slot < num_slots" in msg, msg
    for ok in (-1, 0, 3):
        rc, msg = _call(_exchange(fmt=fmt, wait_slot=ok, num_slots=4), YS)
        assert rc == -1 and "struct_size" in msg, (ok, msg)


def test_too_many_layers_and_null_outputs_are_refused():
    rc, msg = _call(_exchange(n=4), [Y + 0x1000 * l for l in range(5)])
    assert rc == -1 and "VPTQ_MAX_FUSED" in msg, msg
    rc, msg = _call(_exchange(fmt=1), [Y, 0])
    assert rc == -1 and "ys[1] is NULL" in msg, msg


def _c_fields(body):
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        _, names = decl.split(None, 1)            # "<type>[*] name[, name...]" (the header's style)
        for name in names.split(","):
            name = name.strip().lstrip("*")
            out.append((re.match(r"\w+", name).group(0), re.findall(r"\[(\w+)\]", name)))
    return out


def test_exchange_layout_matches_header():
    from vptq_b200 import native
    src = open(os.path.join(ROOT, "include", "vptq_b200.h")).read()
    body = re.search(r"typedef struct vptq_tp_exchange \{(.*?)\} vptq_tp_exchange;", src, re.S).group(1)
    fields = _c_fields(body)
    assert [f for f, _ in fields] == [f for f, _ in native.TpExchange._fields_]
    macros = {k: int(v) for k, v in re.findall(r"#define (VPTQ_\w+) (\d+)\b", src)}
    assert macros["VPTQ_MAX_FUSED"] == native.MAX_FUSED == 4 and macros["VPTQ_MAX_RANKS"] == native.MAX_RANKS == 8
    assert macros["VPTQ_TP_PLAIN"] == native.TP_PLAIN and macros["VPTQ_TP_TAGGED"] == native.TP_TAGGED
    dims = dict(fields)
    assert [macros[d] for d in dims["peer_y"]] == [native.MAX_FUSED, native.MAX_RANKS]
    assert [macros[d] for d in dims["peer_flags"]] == [native.MAX_RANKS]
    # 5 x 4-byte ints, padding, 32 + 8 pointers, 3 pointers, 2 x 4-byte ints
    assert ctypes.sizeof(native.TpExchange) == 24 + 40 * 8 + 3 * 8 + 8 == 376
    assert native.TpExchange.peer_y.offset == 24 and native.TpExchange.format.offset == 368
