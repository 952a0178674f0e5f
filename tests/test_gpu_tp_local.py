"""The tensor-parallel exchange fused into the decode kernels, run on ONE GPU with P virtual ranks.

The kernels only see raw addresses (`peer_y[l][r]`, `peer_flags[r]` of `struct vptq_tp_exchange`): nothing in them
cares whether rank r's buffer lives on another device.  So every virtual rank's full-width activation buffers and
flag array are ordinary allocations on cuda:0 (`LocalArena`), with its own `epoch`, `done` and `error` words, and
the ranks are launched one after another on one stream.  That executes every instruction of the exchange -- the
plain stores and epoch flags, the tagged 8-byte words, `tp_untag`, the host-side exchange checks -- except the
NVLink transport.  It does not exercise concurrency between ranks: `tests/test_gpu_tp.py` (two GPUs) does.

Launch discipline (every test): one stream; for each launch slot, ranks 0 .. P-1, then the next slot.  Virtual
ranks never run on concurrent streams: the list kernel fills every SM, and a consumer spinning on a producer that
cannot be scheduled would only end at the ~2 s timeout.  The eager passes synchronise after every slot and assert
that what the next slot waits for is in place (flags = epoch, tags = run * num_slots + slot + 1) before launching
it, and every exchanged buffer is poisoned first -- NaN, and for the tagged format NaN carrying the tag its consumer
will expect -- so a missing store fails an assert instead of spinning.  No test depends on the timeout firing.
"""
import copy
import functools
import time

import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _util import TOL, parity_error

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
NAN16 = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0}
ZERO = 65536 * 4 + 65536 * 64          # the workspace's zero-at-rest head (DESIGN.md section 1)
M32 = 0xFFFFFFFF


def _i32(v):
    """uint32 value -> the int32 with the same bits (torch stores the counters as int32)."""
    v &= M32
    return v - (1 << 32) if v >= 1 << 31 else v


def _u32(t):
    return t.to(torch.int64) & M32


# ------------------------------------------------------------------------------------------------ layers and oracle
def _key(kw):
    return tuple(sorted(kw.items()))


@functools.lru_cache(maxsize=None)
def _layer(key):
    """(oracle Layer, fp64 W [O][I], fp64 bias or None, full VQuantLinear on cuda:0) -- once per session."""
    from _gpu import make_module
    kw = dict(key)
    L = vo.make_layer(**kw)
    W = vo.dequant(L, out_dtype=np.float64)
    b = None if L.bias is None else vo.to_f32(L.bias, L.dtype).astype(np.float64)
    return L, W, b, make_module(L, DEV)


@functools.lru_cache(maxsize=None)
def _shard_desc(key, rank, world):
    """Descriptor of `rank`'s shard (tp.shard_module), index lists included where the layer is eligible."""
    from vptq_b200 import tp
    L, _, _, full = _layer(key)
    sh = tp.shard_module(full, rank, world).shard
    sh(torch.zeros(0, L.in_features, device=DEV, dtype=full.centroids.weight.dtype))   # builds the descriptor
    d = sh._desc_cache[0]
    d._shard = sh                       # keeps the shard's tensors alive with the descriptor
    return d


def _np64(t):
    """16-bit tensor -> float64 numpy (exact)."""
    t = t.detach().cpu()
    if t.dtype == torch.bfloat16:
        return vo.to_f32(t.view(torch.int16).numpy().view(np.uint16), "bf16").astype(np.float64)
    return t.numpy().astype(np.float64)


def _oracle(key, x):
    _, W, b, _ = _layer(key)
    y = _np64(x) @ W.T
    return y if b is None else y + b[None, :]


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _ws_head_is_zero():
    from vptq_b200 import native
    ws = native.workspace(torch.device(DEV), 0)
    return int(ws[:min(ZERO, ws.numel())].count_nonzero()) == 0


# ------------------------------------------------------------------------------------------------ virtual ranks
class LocalArena:
    """The part of tp.PeerArena that tp.make_exchange uses, with every rank's arena on cuda:0: `world`, `rank`,
    `alloc` (here: every rank's view of the new object) and `peer_ptr`.  `for_rank(r)` is the arena as rank r
    sees it."""

    def __init__(self, world, nbytes):
        self.world, self.rank = world, 0
        self.nbytes = (int(nbytes) + 1023) // 1024 * 1024
        self.bufs = [torch.zeros(self.nbytes, dtype=torch.uint8, device=DEV) for _ in range(world)]
        self.ptrs = [b.data_ptr() for b in self.bufs]
        self._top = 0

    def alloc(self, shape, dtype):
        n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
        off = (self._top + 255) // 256 * 256
        if off + n > self.nbytes:
            raise RuntimeError("LocalArena exhausted")
        self._top = off + n
        return [b[off:off + n].view(dtype).view(*shape) for b in self.bufs], off

    def peer_ptr(self, rank, offset):
        return self.ptrs[rank] + offset

    def for_rank(self, rank):
        v = copy.copy(self)
        v.rank = rank
        return v


class Launch:
    """One launch position (slot) of a token: a fused group of layers reading x from `src` (None: the replicated
    x_in) and writing the full-width buffer `dst` at columns `cols[l]`."""

    def __init__(self, slot, wait, keys, src, dst, cols, x_cols=None):
        self.slot, self.wait, self.keys, self.src, self.dst, self.cols = slot, wait, keys, src, dst, cols
        self.x_cols = x_cols          # in_features: the consumer reads the first x_cols values of src


class Harness:
    """P virtual ranks running a sequence of fused launches per token with the exchange of `fmt`."""

    def __init__(self, world, fmt, dtype, launches, buffers, tokens=1, nslots=None, x_features=None):
        from vptq_b200 import native, tp
        self.world, self.fmt, self.dtype, self.tokens = world, fmt, dtype, tokens
        self.tagged = fmt == native.TP_TAGGED
        self.launches = launches
        self.nslots = nslots or len(launches)
        e = 4 if self.tagged else 2
        total = sum(tokens * n * e + 256 for n in buffers.values()) + self.nslots * world * 4 + 8192
        self.arena = LocalArena(world, total)
        self.buf, self.off, self.local = {}, {}, {}
        for name, n in buffers.items():
            if self.tagged:
                self.buf[name], self.off[name] = self.arena.alloc((tokens, n * 4), torch.uint8)
                self.local[name] = [torch.zeros(tokens, n, dtype=dtype, device=DEV) for _ in range(world)]
            else:
                self.buf[name], self.off[name] = self.arena.alloc((tokens, n), dtype)
                self.local[name] = self.buf[name]
        self.width = dict(buffers)
        self.flags, off_flags = self.arena.alloc((self.nslots, world), torch.int32)
        self.epoch = [torch.zeros(self.nslots, dtype=torch.int32, device=DEV) for _ in range(world)]
        self.done = [torch.zeros(self.nslots, dtype=torch.int32, device=DEV) for _ in range(world)]
        self.error = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(world)]
        self.x_in = torch.zeros(tokens, x_features, dtype=dtype, device=DEV)
        self.fused, self.ex, self.ref, self.ref_ys = [], [], [], []
        for ln in launches:
            per_rank, ex_rank, ref_rank, ys_rank = [], [], [], []
            for r in range(world):
                descs = [_shard_desc(k, r, world) for k in ln.keys]
                o_loc = [d.out_features for d in descs]
                ys = [self.local[ln.dst][r][:, c + r * o:c + (r + 1) * o] for c, o in zip(ln.cols, o_loc)]
                ex = tp.make_exchange(self.arena.for_rank(r), slot=ln.slot, wait_slot=ln.wait,
                                      y_offsets=[self.off[ln.dst] + c * e for c in ln.cols],
                                      slice_bytes=[r * o * e for o in o_loc], flags_offset=off_flags,
                                      epoch=self.epoch[r], done=self.done[r], error=self.error[r],
                                      num_slots=self.nslots, fmt=fmt)
                per_rank.append(native.FusedGemvTP(descs, ys, ex))
                ex_rank.append(ex)
                rys = [torch.zeros(tokens, o, dtype=dtype, device=DEV) for o in o_loc]
                ref_rank.append(native.FusedGemv(descs, rys))
                ys_rank.append(rys)
            self.fused.append(per_rank)
            self.ex.append(ex_rank)
            self.ref.append(ref_rank)
            self.ref_ys.append(ys_rank)

    # -- state
    def set_epochs(self, start):
        """Every slot's epoch at `start` (uint32) and every flag to match, on every rank."""
        for r in range(self.world):
            self.epoch[r].fill_(_i32(start))
            self.flags[r].fill_(_i32(start))

    def runs(self):
        """Current epoch of every slot (uint32), after asserting that all ranks agree."""
        e = [_u32(t).cpu() for t in self.epoch]
        for r in range(1, self.world):
            assert torch.equal(e[r], e[0]), "ranks disagree on the epochs"
        return [int(v) for v in e[0]]

    def tag(self, run, slot):
        return (run * self.nslots + slot + 1) & M32

    # -- buffers
    def values(self, name, r):
        """Rank r's full-width activation buffer as plain 16-bit values [tokens][n]."""
        b = self.buf[name][r]
        if not self.tagged:
            return b
        return b.view(torch.int32).view(self.tokens, -1, 2)[:, :, 0].contiguous().view(self.dtype)

    def tags(self, name, r):
        return _u32(self.buf[name][r].view(torch.int32).view(self.tokens, -1, 2)[:, :, 1])

    def x_of(self, ln, r):
        """What launch `ln` of rank r reads as x (the tagged buffer itself for a tagged consumer)."""
        if ln.src is None:
            return self.x_in
        if self.tagged:
            return self.buf[ln.src][r]
        return self.buf[ln.src][r][:, :ln.x_cols]

    def poison(self, name, tag=None):
        """NaN into every rank's exchanged buffer and local outputs; tagged words carry `tag`, the tag the consumer
        will expect, so a word the producer fails to overwrite is read at once as NaN, never waited on."""
        nan = NAN16[self.dtype]
        for r in range(self.world):
            self.local[name][r].fill_(float("nan"))
            if self.tagged:
                w = self.buf[name][r].view(torch.int32).view(self.tokens, -1, 2)
                w[:, :, 0].fill_(_i32(nan | nan << 16))
                w[:, :, 1].fill_(_i32(tag))

    def poison_token(self, runs):
        first = {}
        for ln in self.launches:
            first.setdefault(ln.dst, ln.slot)
        for name in self.buf:
            s = first.get(name)
            self.poison(name, self.tag(runs[s], s) if s is not None else 0)

    # -- launching
    def launch(self, i, flags):
        for r in range(self.world):
            self.fused[i][r](self.x_of(self.launches[i], r), flags)

    def untag_last(self):
        """tp_untag of the last launch's output on every rank (tagged format): plain copies [tokens][n]."""
        from vptq_b200 import native
        ln = self.launches[-1]
        outs = []
        for r in range(self.world):
            y = torch.full((self.tokens, self.width[ln.dst]), float("nan"), dtype=self.dtype, device=DEV)
            native.tp_untag(self.buf[ln.dst][r], y, self.ex[-1][r])
            outs.append(y)
        return outs

    def consumed_x(self, ln):
        """The x launch `ln` consumed, as plain values (rank 0's copy; the ranks' copies are checked equal)."""
        if ln.src is None:
            return self.x_in
        return self.values(ln.src, 0)[:, :ln.x_cols]

    def check_launch(self, i, run, flags):
        """After slot i ran on every rank (synchronised): the exchange state and the values."""
        ln = self.launches[i]
        want = (run + 1) & M32
        for r in range(self.world):
            assert int(self.error[r].item()) == 0, f"rank {r}: error word set"
            assert int(self.done[r][ln.slot].item()) == 0, f"rank {r}: done counter not back at 0"
            assert int(_u32(self.epoch[r][ln.slot])) == want, f"rank {r} slot {ln.slot}: epoch did not advance"
            if not self.tagged:
                peers = [s for s in range(self.world) if s != r]
                got = _u32(self.flags[r][ln.slot, peers]).cpu().tolist()
                assert got == [want] * len(peers), f"rank {r} slot {ln.slot}: flags {got} != epoch {want}"
        x = self.consumed_x(ln)
        for r in range(self.world):
            self.ref[i][r](self.x_of(ln, r) if ln.src is None else x, flags)
        full = [self.values(ln.dst, r) for r in range(self.world)]
        for k, key in enumerate(ln.keys):
            n = _layer(key)[0].out_features
            c0 = ln.cols[k]
            ref = torch.cat([self.ref_ys[i][r][k] for r in range(self.world)], dim=1)
            y_star = _oracle(key, x)
            for r in range(self.world):
                got = full[r][:, c0:c0 + n]
                assert _same_bits(got, full[0][:, c0:c0 + n]), f"rank {r} layer {k}: buffers differ between ranks"
                assert _same_bits(got, ref), f"rank {r} layer {k}: exchanged values != FusedGemv of the shards"
                if self.tagged:
                    tags = self.tags(ln.dst, r)[:, c0 // 2:(c0 + n) // 2]
                    assert bool((tags == self.tag(run, ln.slot)).all()), f"rank {r} layer {k}: tag missing"
                o = n // self.world
                sl = slice(c0 + r * o, c0 + (r + 1) * o)
                assert _same_bits(self.local[ln.dst][r][:, sl], got[:, r * o:(r + 1) * o]), \
                    f"rank {r} layer {k}: local ys != exchanged values"
            err = parity_error(_np64(full[0][:, c0:c0 + n]), y_star)
            assert err <= TOL[_layer(key)[0].dtype], f"layer {k}: {err:.3e} against the fp64 oracle"

    def eager_token(self, flags):
        """One token, slot by slot, every slot checked before the next one is launched."""
        runs = self.runs()
        self.poison_token(runs)
        for i, ln in enumerate(self.launches):
            if i and any(l2.dst == ln.dst for l2 in self.launches[:i]):
                self.poison(ln.dst, self.tag(runs[ln.slot], ln.slot))   # a buffer written twice per token
            self.launch(i, flags)
            torch.cuda.synchronize()
            self.check_launch(i, runs[ln.slot], flags)
        if self.tagged:
            outs = self.untag_last()
            torch.cuda.synchronize()
            last = self.launches[-1].dst
            for r in range(self.world):
                assert _same_bits(outs[r], self.values(last, r)), f"rank {r}: tp_untag != the last buffer"
        for r in range(self.world):
            assert int(self.error[r].item()) == 0
        assert _ws_head_is_zero(), "workspace not zero at rest"
        return runs


# ------------------------------------------------------------------------------------------------ (a) single launches
LIST = dict(vector_len=8, num_centroids=65536, num_res_centroids=256)
GROUPS = {
    # list kernel (one token): q|k|v-like, K = 8192 without residual codebook, bf16, a 4-layer group with a bias
    "lists_qkv": [dict(in_features=1024, out_features=o, seed=100 + i, **LIST) for i, o in enumerate((1536, 384, 384))],
    "lists_k8192_r0": [dict(in_features=1024, out_features=o, vector_len=8, num_centroids=8192, seed=110 + i)
                       for i, o in enumerate((768, 1152))],
    "lists_bf16": [dict(in_features=2048, out_features=768, dtype="bf16", seed=120, **LIST)],
    "lists_x4_bias": [dict(in_features=1024, out_features=o, bias=i == 1, seed=130 + i, **LIST)
                      for i, o in enumerate((384, 192, 576, 384))],
    # generic kernel (plain format only)
    "generic_k4096": [dict(in_features=1024, out_features=o, vector_len=8, num_centroids=4096, num_res_centroids=256,
                           bias=True, seed=140 + i) for i, o in enumerate((768, 384))],
    "generic_outlier": [dict(in_features=1024 + 128, out_features=768, vector_len=8, num_centroids=4096,
                             num_res_centroids=256, outlier_size=128, outlier_vector_len=4,
                             num_outlier_centroids=4096, bias=True, seed=150)],
}
WORLDS = (1, 2, 3, 4, 8)


def _single(world, fmt, group, tokens):
    specs = GROUPS[group]
    keys = [_key(s) for s in specs]
    cols, c = [], 0
    for s in specs:
        cols.append(c)
        c += s["out_features"]
    dtype = torch.bfloat16 if specs[0].get("dtype") == "bf16" else torch.float16
    h = Harness(world, fmt, dtype, [Launch(0, -1, keys, None, "y", cols)], {"y": c}, tokens=tokens,
                x_features=specs[0]["in_features"])
    x_np = vo.make_x(tokens, specs[0]["in_features"], specs[0].get("dtype", "fp16"), seed=7 + world)
    from _gpu import to_t
    h.x_in.copy_(to_t(x_np, _layer(keys[0])[0], device=DEV))
    return h


CASES_A = [(g, fmt, t) for g in GROUPS for fmt, t in ((0, 1), (1, 1), (0, 2))
           if not (g.startswith("generic") and fmt == 1)]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("group,fmt,tokens", CASES_A,
                         ids=[f"{g}-{'tagged' if f else 'plain'}-t{t}" for g, f, t in CASES_A])
def test_single_launch_exchange(world, group, fmt, tokens):
    """One fused launch per rank (wait_slot -1): every rank's full buffer holds, bit for bit, the concatenation of the
    shards' FusedGemv outputs, within TOL of the fp64 oracle; epoch, done, flags and the workspace as documented."""
    h = _single(world, fmt, group, tokens)
    for _ in range(2):                     # the second token reuses the buffers with advanced epochs
        h.eager_token(0)


# ------------------------------------------------------------------------------------------------ (b) decoder chain
HID, KV, FFN = 1536, 384, 3072


def _chain(world, fmt, dtype=torch.float16, nlayers=2):
    """bench.py:make_step's layout: per decoder layer the launches q|k|v, o, gate|up, down; hidden states ping-pong;
    8 slots per token.  Tagged: every layer K = 65536 (list kernel).  Plain: o and down of the second layer are
    K = 4096 layers, which run the generic kernel."""
    from vptq_b200 import native
    tagged = fmt == native.TP_TAGGED
    dt = "bf16" if dtype == torch.bfloat16 else "fp16"
    launches = []
    for li in range(nlayers):
        def k(name, i, o, seed):
            kw = dict(in_features=i, out_features=o, dtype=dt, seed=1000 * (li + 1) + seed, **LIST)
            if not tagged and li == 1 and name in ("o", "down"):
                kw["num_centroids"] = 4096
            return _key(kw)
        qkv = [k("q", HID, HID, 1), k("k", HID, KV, 2), k("v", HID, KV, 3)]
        hs = f"hs{li % 2}"
        launches += [
            Launch(4 * li, -1 if li == 0 else 4 * li - 1, qkv, None if li == 0 else f"hs{(li - 1) % 2}", "qkv",
                   [0, HID, HID + KV], x_cols=HID),
            Launch(4 * li + 1, 4 * li, [k("o", HID, HID, 4)], "qkv", "o", [0], x_cols=HID),
            Launch(4 * li + 2, 4 * li + 1, [k("gate", HID, FFN, 5), k("up", HID, FFN, 6)], "o", "gu", [0, FFN],
                   x_cols=HID),
            Launch(4 * li + 3, 4 * li + 2, [k("down", FFN, HID, 7)], "gu", hs, [0], x_cols=FFN),
        ]
    bufs = {"qkv": HID + 2 * KV, "o": HID, "gu": 2 * FFN, "hs0": HID, "hs1": HID}
    h = Harness(world, fmt, dtype, launches, bufs, x_features=HID)
    from _gpu import to_t
    L0 = _layer(launches[0].keys[0])[0]
    h.x_in.copy_(to_t(vo.make_x(1, HID, dt, seed=5), L0, device=DEV))
    return h


CASES_B = ([("tagged", torch.float16, w, pdl) for w in WORLDS for pdl in (True, False)] +
           [("plain", torch.float16, w, pdl) for w in WORLDS for pdl in (True, False)] +
           [("tagged", torch.bfloat16, w, pdl) for w, pdl in ((2, True), (3, False))])


@pytest.mark.parametrize("fmt,dtype,world,pdl", CASES_B,
                         ids=[f"{f}-{str(d)[6:]}-w{w}-{'pdl' if p else 'nopdl'}" for f, d, w, p in CASES_B])
def test_decoder_chain(fmt, dtype, world, pdl):
    """Two decoder layers, 5 tokens: every launch against the fp64 oracle on the x it actually consumed and bit for
    bit against FusedGemv on that x; the tagged chain ends with tp_untag, equal to the last buffer."""
    from vptq_b200 import native
    h = _chain(world, native.TP_TAGGED if fmt == "tagged" else native.TP_PLAIN, dtype)
    for t in range(5):
        runs = h.eager_token(native.FLAG_PDL if pdl else 0)
        assert runs == [t] * h.nslots


# ------------------------------------------------------------------------------------------------ (c) graph replay
@pytest.mark.parametrize("fmt,world", [("tagged", 2), ("tagged", 8), ("plain", 3), ("plain", 8)])
def test_graph_replay_of_a_whole_token(fmt, world):
    """All ranks and all slots of one token in one CUDA graph with PDL, replayed 10 times on the same read-only x_in:
    outputs bit-identical to the eager token, epochs and tags advance by one per replay, the error word stays 0."""
    from vptq_b200 import native
    tagged = fmt == "tagged"
    h = _chain(world, native.TP_TAGGED if tagged else native.TP_PLAIN)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        h.eager_token(native.FLAG_PDL)               # (also creates the stream's workspace outside the capture)
        want = {n: [h.values(n, r).clone() for r in range(world)] for n in h.buf}
        last = h.launches[-1].dst
        out = torch.zeros(1, h.width[last], dtype=h.dtype, device=DEV)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for i in range(len(h.launches)):
                h.launch(i, native.FLAG_PDL)
            if tagged:
                native.tp_untag(h.buf[last][0], out, h.ex[-1][0])
        for k in range(10):
            runs = h.runs()
            assert runs == [1 + k] * h.nslots
            h.poison_token(runs)
            out.fill_(float("nan"))
            g.replay()
            s.synchronize()
            for r in range(world):
                assert int(h.error[r].item()) == 0
            assert h.runs() == [2 + k] * h.nslots
            for n in h.buf:
                for r in range(world):
                    assert _same_bits(h.values(n, r), want[n][r]), (k, n, r)
            if tagged:
                assert _same_bits(out, want[last][0])
                for ln in h.launches[-4:]:        # the words last written in this token carry this run's tags
                    for r in range(world):
                        c0, c1 = ln.cols[0], ln.cols[-1] + _layer(ln.keys[-1])[0].out_features
                        assert bool((h.tags(ln.dst, r)[:, c0 // 2:c1 // 2] == h.tag(1 + k, ln.slot)).all())
        assert _ws_head_is_zero()


# ------------------------------------------------------------------------------------------------ (d) counter wrap
@pytest.mark.parametrize("fmt,world", [("plain", 2), ("plain", 3), ("tagged", 2), ("tagged", 4)])
def test_epoch_counters_wrap(fmt, world):
    """Four tokens across the wrap of the 32-bit counters: plain epochs from 2^32 - 2, tagged epochs from
    2^32 // num_slots - 2 (where run * num_slots + slot + 1 wraps), flags set to match.  On one GPU this shows that
    the serial-number flag compare neither over-waits across the wrap nor breaks the tags.  It cannot show the wait
    that the old `flag < want` compare skipped at epoch 2^32 - 1: with sequential virtual ranks every producer has
    finished before its consumer starts, so a skipped wait reads correct data anyway; that needs two GPUs."""
    from vptq_b200 import native
    tagged = fmt == "tagged"
    h = _chain(world, native.TP_TAGGED if tagged else native.TP_PLAIN)
    start = (1 << 32) // h.nslots - 2 if tagged else (1 << 32) - 2
    h.set_epochs(start)
    for t in range(4):
        runs = h.eager_token(native.FLAG_PDL)
        assert runs == [(start + t) & M32] * h.nslots


# ------------------------------------------------------------------------------------------------ (e) refusals
def _call_tp(descs, x, ys, ex, ws, flags=0):
    from vptq_b200 import native
    import ctypes
    n = len(descs)
    darr = (ctypes.POINTER(native.LinearDesc) * n)(*[ctypes.pointer(d) for d in descs])
    yarr = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
    sarr = (ctypes.c_int64 * n)(*[y.stride(0) for y in ys])
    wp, wb = (ws.data_ptr(), ws.numel()) if ws is not None else (None, 0)
    rc = native.lib().vptq_b200_quant_gemv_multi_tp(n, darr, x.data_ptr(), native.row_pitch(x), yarr, sarr,
                                                    x.shape[0], ctypes.byref(ex), wp, wb, flags,
                                                    torch.cuda.current_stream().cuda_stream)
    native.check(rc, "vptq_b200_quant_gemv_multi_tp")


def _refusal_case(world, fmt, keys, tokens, ws_mode, match):
    from vptq_b200 import native
    L0 = _layer(keys[0])[0]
    dtype = torch.float16
    cols, c = [], 0
    for k in keys:
        cols.append(c)
        c += _layer(k)[0].out_features
    h = Harness(world, fmt, dtype, [Launch(0, -1, keys, None, "y", cols)], {"y": c}, tokens=tokens,
                x_features=L0.in_features)
    from _gpu import to_t
    h.x_in.copy_(to_t(vo.make_x(tokens, L0.in_features, "fp16", seed=3), L0, device=DEV))
    h.poison_token(h.runs())
    torch.cuda.synchronize()
    before = [[_bits(y).clone() for y in f.ys] for f in h.fused[0]]
    ws = native.workspace(torch.device(DEV), sum(native.workspace_bytes(_shard_desc(k, 0, world), tokens,
                                                                        native.OP_GEMV) for k in keys))
    for r in range(world):
        f = h.fused[0][r]
        with pytest.raises(RuntimeError, match=match):
            if ws_mode == "none":
                _call_tp(f.descs, h.x_in, f.ys, f.ex, None)
            else:
                f(h.x_in)
    torch.cuda.synchronize()
    for r in range(world):
        assert torch.equal(_u32(h.epoch[r]), torch.zeros_like(_u32(h.epoch[r]))), "epoch moved"
        assert int(h.error[r].item()) == 0 and int(h.done[r].sum().item()) == 0
        for y, b in zip(h.fused[0][r].ys, before[r]):
            assert torch.equal(_bits(y), b), "a refused launch wrote its outputs"


TAGGED_GENERIC = "the tagged exchange format is implemented by the list kernel only"


@pytest.mark.parametrize("world", [1, 2, 4])
def test_tagged_format_refused_on_the_generic_route(world):
    """Tagged needs the list kernel: two tokens, layers without lists, or no workspace are refused loudly, at every
    world size (world 1 included), and nothing is written."""
    from vptq_b200 import native
    lists = [_key(GROUPS["lists_qkv"][0])]
    _refusal_case(world, native.TP_TAGGED, lists, 2, "ws", TAGGED_GENERIC)
    _refusal_case(world, native.TP_TAGGED, [_key(s) for s in GROUPS["generic_k4096"]], 1, "ws", TAGGED_GENERIC)
    _refusal_case(world, native.TP_TAGGED, lists, 1, "none", TAGGED_GENERIC)


@pytest.mark.parametrize("world", [1, 2])
def test_layers_the_fused_generic_kernel_refuses(world):
    """v != 8 and a 16-group layer (the global split-K route) cannot run inside the exchange: refused, nothing
    written, epochs unchanged."""
    from vptq_b200 import native
    v4 = _key(dict(in_features=1024, out_features=512, vector_len=4, num_centroids=4096, seed=160))
    g16 = _key(dict(in_features=4096, out_features=512, vector_len=8, num_centroids=256, num_codebooks=16, seed=161))
    _refusal_case(world, native.TP_PLAIN, [v4], 1, "ws", "vector_len 8")
    _refusal_case(world, native.TP_PLAIN, [g16], 1, "ws", "one launch configuration")


# ------------------------------------------------------------------------------------------------ (f) the error word
def test_generic_flag_wait_returns_at_once_when_the_error_word_is_set():
    """Rank 0's generic-route plain consumer whose producer flags were never set, with error = 1 preset: it must not
    wait (the header promises that later waits return at once once the error word is set)."""
    from vptq_b200 import native
    key = _key(GROUPS["generic_k4096"][0])
    L = _layer(key)[0]
    h = Harness(2, native.TP_PLAIN, torch.float16, [Launch(0, -1, [key], None, "a", [0]),
                                                    Launch(1, 0, [key], "a", "b", [0], x_cols=L.in_features)],
                {"a": L.in_features, "b": L.out_features}, x_features=L.in_features)
    h.error[0].fill_(1)
    h.local["a"][0].zero_()
    h.ref[1][0](h.x_of(h.launches[1], 0))      # the same kernel without an exchange: loaded before the clock starts
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    h.fused[1][0](h.x_of(h.launches[1], 0))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert int(h.error[0].item()) == 1
    assert dt < 0.5, f"the consumer waited {dt:.2f} s for flags with the error word set"


# ------------------------------------------------------------------------------------------------ (g) sharded modules
SHARDED = {
    "lists": dict(in_features=1024, out_features=1024, seed=170, **LIST),
    "outlier_bias": dict(in_features=1024 + 128, out_features=512, vector_len=8, num_centroids=4096,
                         num_res_centroids=256, outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096,
                         bias=True, seed=5),
    "groups4": dict(in_features=1024, out_features=512, vector_len=8, num_centroids=4096, num_codebooks=4, seed=171),
}


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", sorted(SHARDED))
def test_sharded_module_slices_sum_to_the_layer(name, world):
    """What TPVQuantLinear's all_reduce mode does before the collective: each rank writes its shard into its column
    slice of a zeroed full-width y; the sum over ranks is the unsharded layer (1, 2 and 40 tokens)."""
    from _gpu import to_t
    from vptq_b200 import native
    key = _key(SHARDED[name])
    L = _layer(key)[0]
    for tokens in (1, 2, 40):
        x_np = vo.make_x(tokens, L.in_features, L.dtype, seed=tokens)
        x = to_t(x_np, L, device=DEV)
        total = torch.zeros(tokens, L.out_features, dtype=torch.float32, device=DEV)
        o = L.out_features // world
        for r in range(world):
            y = torch.zeros(tokens, L.out_features, dtype=x.dtype, device=DEV)
            (native.quant_gemv if tokens < 3 else native.quant_gemm)(_shard_desc(key, r, world), x,
                                                                      y[:, r * o:(r + 1) * o])
            total += y.float()
        torch.cuda.synchronize()
        err = parity_error(total.cpu().numpy(), _oracle(key, x))
        assert err <= TOL[L.dtype], (name, world, tokens, err)


# ------------------------------------------------------------------------------------------------ (h) expanded x
@pytest.mark.parametrize("group", ["lists_qkv", "generic_k4096"])
def test_fused_tp_takes_a_one_row_expanded_x(group):
    """FusedGemvTP with a one-row x made by `expand` (row stride 0), as every other entry point accepts it: the same
    bits as the contiguous x."""
    from vptq_b200 import native
    h = _single(2, native.TP_PLAIN, group, 1)
    h.eager_token(0)
    want = [h.values("y", r).clone() for r in range(2)]
    row = h.x_in[0].clone()
    xe = row.expand(2, row.shape[0])[:1]       # (torch gives a fresh size-1 dimension a nonzero stride)
    assert xe.shape[0] == 1 and xe.stride(0) == 0
    h.poison_token(h.runs())
    for r in range(2):
        h.fused[0][r](xe)
    torch.cuda.synchronize()
    for r in range(2):
        assert _same_bits(h.values("y", r), want[r])
