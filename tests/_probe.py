"""Basis-probe helpers: the exact per-column answer of every kernel route, and the tools the probe tests use.

With x = e_f (1.0 at input feature f, 0 elsewhere) every output is a single product, so the value a kernel
returns is fixed to the last bit by its documented arithmetic.  `probe_expect(L, route)` simulates that
arithmetic in numpy (float32 operations are IEEE round-to-nearest, like the GPU's) and returns [I, O]: row f
is the output of the probe e_f, rounded to the layer's 16-bit type.

  route      kernel(s)                                        y[o] for x = e_f (cr = C + R in fp32)
  generic    gemv_kernel (any token count)                    rn16(((cr * s) + wb) + bias)
  direct     dequant_o8_kernel + gemm_tn_wgmma                rn16(rn16(fma(cr, s, wb)) + bias)
  prep       prefill_prep_x + dequant_q8/dequant_kernel + GEMM rn16(((s * rn16(C + R)) + wb) + bias)
  lists      gemv_lists_kernel (one token)                    2^-30 fixed-point sum, see _lists_fixed()

s = weight_scale[f], wb = weight_bias[f] (1 and 0 without norm); every operator rounds to fp32 once.
"""
import re
import time

import numpy as np
import torch

import vptq_oracle as vo

ROUTES = ("generic", "direct", "prep", "lists")
_FIX = 2.0 ** 30


def _f32(a):
    return np.asarray(a, dtype=np.float32)


def _fp16(a):
    """round to fp16, returned as fp32 (numpy's float64/float32 -> float16 casts round to nearest even)"""
    return np.asarray(a).astype(np.float16).astype(np.float32)


def _perm_inverse(L):
    if L.perm is None:
        return None
    return np.argsort(np.asarray(L.perm).astype(np.uint16).astype(np.int64), kind="stable")


def _column_terms(L, o, idx, ridx):
    """C, R (fp32 of the 16-bit entries) and the codebook slice of output rows `o`, columns in ORIGINAL order.
    Outlier columns carry their codebook value in C and zero in R."""
    v, G = L.vector_len, L.num_codebooks
    C = vo.to_f32(L.centroids, L.dtype).reshape(G, L.num_centroids, v)
    r, e = o // v, (o % v)[:, None]
    main = np.concatenate([C[g][idx[g][r], e] for g in range(G)], axis=1)
    sl = np.concatenate([idx[g][r] >> 12 for g in range(G)], axis=1)
    if L.res_bits:
        R = vo.to_f32(L.res_centroids, L.dtype).reshape(G, L.num_res_centroids, v)
        res = np.concatenate([R[g][ridx[g][r], e] for g in range(G)], axis=1)
    else:
        res = np.zeros_like(main)
    if L.enable_outlier:
        vol, S = L.outlier_vector_len, L.outlier_size
        Col = vo.to_f32(L.outlier_centroids, L.dtype).reshape(L.num_outlier_centroids, vol)
        oidx = np.asarray(L.outlier_indices).astype(np.uint16).astype(np.int64).reshape(-1, S)
        wo = Col[oidx[o // vol], (o % vol)[:, None]]
        main = np.concatenate([wo, main], axis=1)
        res = np.concatenate([np.zeros_like(wo), res], axis=1)
        sl = np.concatenate([np.zeros(wo.shape, dtype=sl.dtype), sl], axis=1)
    inv = _perm_inverse(L)
    if inv is not None:
        main, res, sl = main[:, inv], res[:, inv], sl[:, inv]
    return main, res, sl


def _lists_fixed(p, wb, sl, has_norm):
    """The list kernel's reduction: every unit converts its fp32 sum to 2^-30 fixed point (round to nearest even)
    and adds it into a 64-bit accumulator.  The weight_bias term of a column tile is added, in fp32, to the sum of
    that tile's slice-0 unit; the probe's own term sits in the unit of its codebook slice."""
    if not has_norm:
        return np.rint(p.astype(np.float64) * _FIX)
    same = np.rint((p + wb).astype(np.float64) * _FIX)
    apart = np.rint(p.astype(np.float64) * _FIX) + np.rint(wb.astype(np.float64) * _FIX)
    return np.where(sl == 0, same, apart)


def probe_expect(L, route, block_rows=2048):
    """[I, O] float32: row f = the 16-bit output of `route` for the probe x = e_f (see the module docstring)."""
    if route not in ROUTES:
        raise ValueError(route)
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    I, O, dt = L.in_features, L.out_features, L.dtype
    has_norm = L.weight_scale is not None
    s = vo.to_f32(L.weight_scale, dt) if has_norm else np.ones(I, np.float32)
    wb = vo.to_f32(L.weight_bias, dt) if has_norm else np.zeros(I, np.float32)
    bias = vo.to_f32(L.bias, dt) if L.bias is not None else None
    out = np.empty((O, I), dtype=np.float32)
    for o0 in range(0, O, block_rows):
        o = np.arange(o0, min(O, o0 + block_rows))
        main, res, sl = _column_terms(L, o, idx, ridx)
        if route == "generic":
            y = _f32(main + res) * s
            if has_norm:
                y = y + wb
        elif route == "direct":
            w = (main.astype(np.float64) + res) * s + wb          # exact: fma(cr, s, wb) rounds once, below
            y = vo.round_to(_f32(w), dt)
        elif route == "prep":
            c16 = vo.round_to(_f32(main.astype(np.float64) + res), dt)
            y = s * c16                                            # exact in fp32 (two 16-bit factors)
            if has_norm:
                y = y + wb
        else:
            if dt == "fp16":   # x' = x * s in fp16 (exact), c + r in packed fp16
                xq, c = s, _fp16(main.astype(np.float64) + res)
            else:              # x' = x * s in bf16 (exact), c + r in fp32
                xq, c = s, _f32(main + res)
            p = _f32(c.astype(np.float64) * xq)
            q = _lists_fixed(p, wb, sl, has_norm)
            y = _f32(q) * np.float32(1.0 / _FIX)
        if bias is not None:
            y = y + bias[o][:, None]
        out[o] = vo.round_to(_f32(y), dt)
    return np.ascontiguousarray(out.T)


def fp64_weight(L, device="cuda"):
    """The layer's dense weight [O, I] in float64 on `device`: y* = x.double() @ W64.T (+ bias)."""
    return torch.from_numpy(vo.dequant(L, np.float64)).to(device)


def fp64_bias(L, device="cuda"):
    return None if L.bias is None else torch.from_numpy(vo.to_f32(L.bias, L.dtype).astype(np.float64)).to(device)


def launched_kernels(fn):
    """Names of the CUDA kernels that one call of `fn` launched (torch.profiler, CUPTI).

    The profiler maps GPU timestamps onto the host clock and keeps only records inside the session; late in a long
    process the mapped times drift, and records at either end of a short session fall outside it.  So `fn` runs
    between two marker kernels, `lead` seconds inside both ends of the session: when both markers are recorded,
    everything `fn` launched between them is too.  Otherwise the call is repeated with a longer lead."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    marker = torch.zeros(1, dtype=torch.int64, device="cuda")
    for lead in (0.0, 0.05, 0.25, 1.0, 4.0):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            time.sleep(lead)
            marker.add_(1)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            marker.add_(1)
            torch.cuda.synchronize()
            time.sleep(lead)
        # the raw activity records: the FunctionEvent tree built from them can drop kernels that no torch op launched
        names = [e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == DeviceType.CUDA]
        is_marker = ["CUDAFunctorOnSelf_add<long>" in n for n in names]
        if sum(is_marker) == 2:
            return [n for n, mk in zip(names, is_marker) if not mk]
    raise AssertionError(f"torch.profiler did not record both marker kernels: the route cannot be asserted ({names})")


def ran(names, kernel):
    """Did a kernel named `kernel` (whole identifier, any template arguments) run?"""
    pat = re.compile(r"(?<![A-Za-z0-9_])" + re.escape(kernel) + r"(?![A-Za-z0-9_])")
    return any(pat.search(n) for n in names)


def aligned_rows(n, I, dtype, pitch=None, offset=0, device="cuda"):
    """[n, I] zero view into a larger buffer with row pitch `pitch` (default: I rounded up to 8 elements, so every
    row is 16-byte aligned) starting `offset` elements into it (a fresh allocation is 512-byte aligned)."""
    pitch = pitch if pitch is not None else (I + 7) // 8 * 8
    buf = torch.zeros(offset + max(n - 1, 0) * pitch + I + 64, dtype=dtype, device=device)
    return buf.as_strided((n, I), (pitch, 1), offset)


def _key16(t):
    """16-bit floats -> integers ordered like their values (+0 and -0 both 0): ulp distance = key difference"""
    b = t.contiguous().view(torch.int16).to(torch.int32)
    mag = b & 0x7FFF
    return torch.where(b < 0, -mag, mag)


def ulp_diff(y, expect):
    """|y - expect| in units of the 16-bit type's last place, element-wise (both the same 16-bit dtype)."""
    assert y.dtype == expect.dtype and y.dtype in (torch.float16, torch.bfloat16)
    return (_key16(y) - _key16(expect)).abs()


def to_dev(a, L, device="cuda"):
    """fp32 numpy values that are exact in the layer's 16-bit type -> that 16-bit type on `device`."""
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device).to(dt)
