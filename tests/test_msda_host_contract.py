"""The MSDA host contract without a GPU, over one table of call geometries:

* the exact bytes every MSDA workspace query returns, and the INT8 format answer of b200_msda_supports_format (these
  never touch a device, so they run everywhere);
* the status every MSDA entry returns on each geometry and on null, misaligned or out-of-range arguments.

The entries get fabricated device addresses. An entry that accepted one of these rows would launch a kernel on them,
so the status table runs only where no CUDA device is present: there, an accepted row returns B200_ERR_LAUNCH (3)
from its first launch (or from the first runtime call before it), and a rejected row (1 or 2) must not have counted a
launch.
"""
import ctypes

import pytest
import torch

from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.workloads import CONFIGS

# The C ABI's argument order: batch, spatial_size, num_heads, channels, num_levels, num_query, num_point,
# points_per_group.
GEO = {
    name: (c.batch, c.spatial_size, c.num_heads, c.channels, c.num_levels, c.num_query, c.num_points, c.points_per_group)
    for name, c in CONFIGS.items()
}
_BASE = GEO["small_sca"]


def _edit(**kw):
    keys = ("B", "S", "M", "C", "L", "Q", "P", "G")
    return tuple(kw.get(k, v) for k, v in zip(keys, _BASE))


GEO.update({
    # every dimension at 0
    "B0": _edit(B=0), "S0": _edit(S=0), "M0": _edit(M=0), "C0": _edit(C=0),
    "L0": _edit(L=0), "Q0": _edit(Q=0), "P0": _edit(P=0), "G0": _edit(G=0),
    # levels around the packed INT8 kernel's 8 and the 16 every kernel takes
    "L8": _edit(L=8, P=4), "L9": _edit(L=9, P=4), "L16": _edit(L=16, P=4), "L17": _edit(L=17, P=4),
    # points per item (L * P) around the kernels' bounds: the packed INT8 kernel's 16 and 32, the resident-tail
    # kernel's 32, the backward's 64, the forward's 64 chunks of 4
    "LP12": _edit(L=3, P=4), "LP15": _edit(L=3, P=5), "LP16": _edit(L=4, P=4), "LP32": _edit(L=2, P=16),
    "LP33": _edit(L=3, P=11), "LP64": _edit(L=4, P=16), "LP65": _edit(L=5, P=13), "LP128": _edit(L=4, P=32),
    "LP256": _edit(L=16, P=16), "LP260": _edit(L=13, P=20),
    "C30": _edit(C=30), "C31": _edit(C=31), "C64": _edit(C=64),
    "P6": _edit(P=6), "G2": _edit(G=2), "G3": _edit(G=3),
    "M64": _edit(M=64),  # the INT8 pack tile no longer fits shared memory
    # (S + 1) * M * C * 4 just below and at 2^31
    "S_max": _edit(S=(1 << 31) // (8 * 32 * 4) - 2), "S_over": _edit(S=(1 << 31) // (8 * 32 * 4) - 1),
    "BS_over": _edit(B=8000, S=300000),  # B * S >= 2^31: the resident-tail kernel's row count
    "slab_over": _edit(M=1, S=12000000, L=4, P=4),  # 3 * S * 64 >= 2^31: the packed INT8 kernel's slab offsets
})


def _enqueue_descs(geo, dtype, ref_dtype=None, scale_o=0.5):
    """The five input descriptors and the output descriptor TensorRT would pass to b200_msda_enqueue for `geo`."""
    b, s, m, c, l, q, p, g = geo
    shapes = [(b, s, m, c), (l, 2), (b, q, 1, 2 * g), (b, q, m, l * p * 2), (b, q, m, l * p)]
    types = [dtype, 3, dtype if ref_dtype is None else ref_dtype, dtype, dtype]
    ins = (_lib.TensorDesc * 6)()  # io[5] is the output, for b200_msda_supports_format
    for d, sh, t in zip(ins, shapes, types):
        d.dims.nbDims = len(sh)
        d.dims.d[: len(sh)] = sh
        d.type, d.format, d.scale = t, 0, 0.05
    ins[5].dims.nbDims = 3
    ins[5].dims.d[:3] = (b, q, m * c)
    ins[5].type, ins[5].format, ins[5].scale = dtype, 0, scale_o
    return ins


# ---- workspace queries ---------------------------------------------------------------------------------------------------
WS_COLUMNS = ("i8", "bw_f32", "bw_f16", "bw_bf16", "bw_2", "enq_f32", "enq_f16", "enq_i8", "fmt_i8")


def workspace_row(geo):
    lib = _lib.load()
    b, s, m, c, l, q, p, g = geo
    row = [lib.b200_msda_i8_workspace_size(b, s, m, c, l, p, g)]
    row += [lib.b200_msda_backward_workspace_size(d, *geo) for d in (0, 1, 7, 2)]
    row += [lib.b200_msda_enqueue_workspace_size(_enqueue_descs(geo, t)) for t in (0, 1, 2)]
    row.append(lib.b200_msda_supports_format(0, _enqueue_descs(geo, 2, 1), 5, 1))
    return dict(zip(WS_COLUMNS, row))


WS = {
    "cpu_plumbing": (0, 6400, 4200704, 4200704, 0, 0, 0, 0, 1),
    "tiny_sca": (0, 3840000, 6144000, 6144000, 0, 0, 0, 0, 1),
    "base_sca": (284083200, 61440000, 250828800, 250828800, 0, 0, 0, 284083200, 1),
    "base_tsa": (0, 5120000, 87040000, 87040000, 0, 0, 0, 0, 1),
    "base_decoder": (0, 57600, 41017600, 41017600, 0, 0, 0, 0, 1),
    "small_sca": (986112, 170496, 827904, 827904, 0, 0, 0, 986112, 1),
    "B0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "S0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "M0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "C0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "L0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "Q0": (986112, 0, 0, 0, 0, 0, 0, 986112, 1),
    "P0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "G0": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "L8": (986112, 170496, 827904, 827904, 0, 0, 0, 986112, 1),
    "L9": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "L16": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "L17": (0, 0, 0, 0, 0, 0, 0, 0, 1),
    "LP12": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "LP15": (0, 170496, 827904, 827904, 0, 0, 0, 0, 0),
    "LP16": (986112, 170496, 827904, 827904, 0, 0, 0, 986112, 1),
    "LP32": (986112, 170496, 827904, 827904, 0, 0, 0, 986112, 1),
    "LP33": (0, 170496, 827904, 827904, 0, 0, 0, 0, 0),
    "LP64": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "LP65": (0, 170496, 827904, 827904, 0, 0, 0, 0, 0),
    "LP128": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "LP256": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "LP260": (0, 170496, 827904, 827904, 0, 0, 0, 0, 1),
    "C30": (0, 170496, 786944, 786944, 0, 0, 0, 0, 0),
    "C31": (0, 170496, 807424, 807424, 0, 0, 0, 0, 0),
    "C64": (0, 170496, 1485312, 1485312, 0, 0, 0, 0, 1),
    "P6": (0, 170496, 827904, 827904, 0, 0, 0, 0, 0),
    "G2": (986112, 85248, 742656, 742656, 0, 0, 0, 986112, 1),
    "G3": (0, 128000, 785408, 785408, 0, 0, 0, 0, 1),
    "M64": (7888896, 1363968, 6623232, 6623232, 0, 0, 0, 7888896, 1),
    "S_max": (6442444800, 170496, 4295133696, 4295133696, 0, 0, 0, 6442444800, 1),
    "S_over": (6442447872, 0, 0, 0, 0, 0, 0, 6442447872, 1),
    "BS_over": (3686400000000, 681984000, 2458281984000, 2458281984000, 0, 0, 0, 3686400000000, 1),
    "slab_over": (4608000000, 21504, 3072021504, 3072021504, 0, 0, 0, 4608000000, 1),
}  # fmt: skip


@pytest.mark.parametrize("name", list(GEO))
def test_workspace_bytes(name):
    assert workspace_row(GEO[name]) == dict(zip(WS_COLUMNS, WS[name]))


# ---- entry status --------------------------------------------------------------------------------------------------------
_A = 1 << 20
_NSLOTS = 13


def _ptrs():
    return [_A * (i + 1) for i in range(_NSLOTS)]  # fabricated 256-byte-aligned device addresses, never dereferenced


# Pointer slots: value 0, spatial_shapes 1, reference_points 2, sampling_offsets 3, attn_weight 4, out / accum / slots /
# grad_output / grad_slots 5, bev_mask 6, records 7, workspace 8, grad_value 9, grad_reference_points 10,
# grad_sampling_offsets 11, grad_attn_weight 12. An entry ignores the slots it has no argument for.
FWD = ("f32", "f16", "f16_h2", "bf16")
SCA = ("sca_f32", "sca_f16", "sca_bf16", "sca_shared_f32", "sca_shared_f16", "sca_shared_bf16")
TRACE = ("f32_trace", "f16_trace", "bf16_trace")
BW = ("backward_f32", "backward_f16", "backward_bf16")
BW_SCA = ("sca_backward_f32", "sca_backward_f16", "sca_backward_bf16", "sca_shared_backward_f32",
          "sca_shared_backward_f16", "sca_shared_backward_bf16")  # fmt: skip
ENQ = {"enq_f32": (0, 0, 0), "enq_f16": (1, 1, 0), "enq_f16_h2": (1, 1, 1), "enq_i8": (2, 1, 0), "enq_i8_ref32": (2, 0, 0)}
ENTRIES = (*FWD, "f16_res", "i8", *SCA, *TRACE, "i8_trace", "i8_ws", "dbg_f32", "dbg_f16", "dbg_2", *BW, *BW_SCA, *ENQ)


def _call(entry, geo, p, scale_o=0.5, ref_half=0, ws_short=False):
    lib = _lib.load()
    b, s, m, c, l, q, n, g = geo
    if entry in FWD:
        return getattr(lib, "b200_msda_" + entry)(*p[:5], *geo, p[5], None)
    if entry == "f16_res":  # b200_msda_f16 with the resident-tail kernel selected
        before = lib.b200_msda_set_f16_path(1)
        try:
            return lib.b200_msda_f16(*p[:5], *geo, p[5], None)
        finally:
            lib.b200_msda_set_f16_path(before)
    i8_head = (p[0], 0.1, p[1], p[2], ref_half, p[3], 0.1, p[4], 0.1)
    if entry == "i8":
        return lib.b200_msda_i8(*i8_head, *geo, p[5], scale_o, None)
    if entry == "i8_trace":
        return lib.b200_msda_i8_trace(*i8_head, *geo, p[5], scale_o, p[7], None)
    if entry == "i8_ws":
        ws = lib.b200_msda_i8_workspace_size(b, s, m, c, l, n, g) - (1 if ws_short else 0)
        return lib.b200_msda_i8_ws(*i8_head, *geo, p[5], scale_o, p[8], max(ws, 0), None, None)
    if entry in SCA:
        return getattr(lib, "b200_msda_" + entry)(*p[:5], p[6], *geo, p[5], None)
    if entry in TRACE:
        return getattr(lib, "b200_msda_" + entry)(*p[:5], *geo, p[5], p[7], None)
    if entry.startswith("dbg_"):
        dtype = {"dbg_f32": 0, "dbg_f16": 1, "dbg_2": 2}[entry]
        return lib.b200_msda_debug_indices(dtype, p[1], p[2], p[3], b, m, l, q, n, g, p[7], None)
    if entry in BW:
        return getattr(lib, "b200_msda_" + entry)(*p[:6], *p[9:13], p[8], *geo, None)
    if entry in BW_SCA:
        return getattr(lib, "b200_msda_" + entry)(*p[:5], p[6], p[5], *p[9:13], p[8], *geo, None)
    dtype, ref_dtype, use_h2 = ENQ[entry]
    io = _enqueue_descs(geo, dtype, ref_dtype, scale_o)
    inputs, outputs = (ctypes.c_void_p * 5)(*p[:5]), (ctypes.c_void_p * 1)(p[5])
    return lib.b200_msda_enqueue(io, ctypes.pointer(io[5]), inputs, outputs, p[8], None, use_h2)


def _case(case):
    """(geometry, pointers, keyword arguments) of a status row: a GEO name, or a change to the "small_sca" call."""
    ptrs, kw = _ptrs(), {}
    if case in GEO:
        return GEO[case], ptrs, kw
    what, _, arg = case.partition(":")
    if what == "null":
        ptrs[int(arg)] = None
    elif what == "shift":  # "shift:<slot>+<bytes>"
        slot, nbytes = map(int, arg.split("+"))
        ptrs[slot] += nbytes
    elif what == "scale_o":
        kw["scale_o"] = float(arg)
    elif what == "C30_scale_o":  # the channel rule and the scale rule broken together
        kw["scale_o"] = float(arg)
        return GEO["C30"], ptrs, kw
    elif what == "ref_half":
        kw["ref_half"] = 1
    elif what == "ws_short":
        kw["ws_short"] = True
    return _BASE, ptrs, kw


def status(entry, case):
    geo, ptrs, kw = _case(case)
    before = _lib.launch_count()
    st = _call(entry, geo, ptrs, **kw)
    if st in (1, 2):
        assert _lib.launch_count() == before, "a rejected call counted a launch"
    return st


POINTER_CASES = [f"null:{i}" for i in range(_NSLOTS)] + [f"shift:{i}+{b}" for i in range(_NSLOTS) for b in (2, 4, 8)]
_SCALE = ["scale_o:0", "scale_o:-1", "scale_o:nan", "C30_scale_o:0"]
EXTRA_CASES = {"i8": _SCALE + ["ref_half"], "i8_trace": _SCALE + ["ref_half"], "i8_ws": _SCALE + ["ref_half", "ws_short"],
               "enq_i8": _SCALE, "enq_i8_ref32": _SCALE}  # fmt: skip
CASES = list(GEO) + POINTER_CASES + sorted({c for cs in EXTRA_CASES.values() for c in cs})


def status_row(case):
    """One character per entry of ENTRIES: its status, or "-" where the case does not apply to it."""
    extra = case in CASES[len(GEO) + len(POINTER_CASES):]
    return "".join("-" if extra and case not in EXTRA_CASES.get(e, ()) else str(status(e, case)) for e in ENTRIES)


# One column per entry of ENTRIES:
#   f32 f16 f16_h2 bf16 f16_res i8 | sca_f32 sca_f16 sca_bf16 sca_shared_f32 sca_shared_f16 sca_shared_bf16 |
#   f32_trace f16_trace bf16_trace i8_trace i8_ws | dbg_f32 dbg_f16 dbg_2 | backward_f32 backward_f16 backward_bf16 |
#   sca_backward_f32 _f16 _bf16 sca_shared_backward_f32 _f16 _bf16 | enq_f32 enq_f16 enq_f16_h2 enq_i8 enq_i8_ref32
# 0 = B200_OK (no gradient requested), 1 = B200_ERR_UNSUPPORTED, 2 = B200_ERR_BAD_PARAM, 3 = accepted (the first launch
# fails without a device).
STATUS = {
    "cpu_plumbing":  "3333333333333333133133333333333333",
    "tiny_sca":      "3333333333333333133133333333333333",
    "base_sca":      "3333333333333333333133333333333333",
    "base_tsa":      "3333333333333333133133333333333333",
    "base_decoder":  "3333333333333333133133333333333333",
    "small_sca":     "3333333333333333333133333333333333",
    "B0":            "2222222222222222222222222222222222",
    "S0":            "2222222222222222233122222222222222",
    "M0":            "2222222222222222222222222222222222",
    "C0":            "2222222222222222133122222222222222",
    "L0":            "2222222222222222122222222222222222",
    "Q0":            "2222222222222222222222222222222222",
    "P0":            "2222222222222222122222222222222222",
    "G0":            "2222222222222222133122222222222222",
    "L8":            "3333333333333333333133333333333333",
    "L9":            "3333333113113333133133333333333333",
    "L16":           "3333333113113333133133333333333333",
    "L17":           "1111111111111111133111111111111111",
    "LP12":          "3333333333333333133133333333333333",
    "LP15":          "3333311111113331133133311111133311",
    "LP16":          "3333333333333333333133333333333333",
    "LP32":          "3333333333333333333133333333333333",
    "LP33":          "3333311111113331133133311111133311",
    "LP64":          "3333333113113333133133333333333333",
    "LP65":          "3333311111113331133133311111133311",
    "LP128":         "3333331111113333133133311111133333",
    "LP256":         "3333331111113333133133311111133333",
    "LP260":         "3333331111113333133133311111133333",
    "C30":           "3333311111113331133133311111133311",
    "C31":           "3313311111113331133133311111133311",
    "C64":           "3333331111113333133133311111133333",
    "P6":            "3333311111113331133133311111133311",
    "G2":            "3333333333333333333133333333333333",
    "G3":            "3333331111113333133133311111133333",
    "M64":           "3333333333333333133133333333333333",
    "S_max":         "3333333333333333333133333333333333",
    "S_over":        "2222222222222222333122222222222233",
    "BS_over":       "3333333333333333333133333333333333",
    "slab_over":     "3333333333333333133133333333333333",
    "null:0":        "2222222222222222233122222222222222",
    "null:1":        "2222222222222222222222222222222222",
    "null:2":        "2222222222222222222222222222222222",
    "null:3":        "2222222222222222222222222222222222",
    "null:4":        "2222222222222222233122222222222222",
    "null:5":        "2222222222222222233122222222222222",
    "null:6":        "3333332222223333333133322222233333",
    "null:7":        "3333333333332222322233333333333333",
    "null:8":        "3333333333333333233122222222233333",
    "null:9":        "3333333333333333333133333333333333",
    "null:10":       "3333333333333333333133333333333333",
    "null:11":       "3333333333333333333133333333333333",
    "null:12":       "3333333333333333333133333333333333",
    "shift:0+2":     "3333331111113333133123321121133333",
    "shift:0+4":     "3333331111113333133133311111133333",
    "shift:0+8":     "3333331111113333133133311111133333",
    "shift:1+2":     "3333331111113333133122222222233333",
    "shift:1+4":     "3333331111113333333133333333333333",
    "shift:1+8":     "3333333333333333333133333333333333",
    "shift:2+2":     "3333331111113333133123221221233333",
    "shift:2+4":     "3333331111113333133133311111133333",
    "shift:2+8":     "3333331111113333133133311111133333",
    "shift:3+2":     "3333331111113333133123321121133333",
    "shift:3+4":     "3333331111113333133133311111133333",
    "shift:3+8":     "3333331111113333133133311111133333",
    "shift:4+2":     "3333331111113333133123321121133333",
    "shift:4+4":     "3333331111113333133133311111133333",
    "shift:4+8":     "3333331111113333133133311111133333",
    "shift:5+2":     "3333331111113333133123322222233333",
    "shift:5+4":     "3333331111113333133133311111133333",
    "shift:5+8":     "3333331111113333133133311111133333",
    "shift:6+2":     "3333333333333333333133322222233333",
    "shift:6+4":     "3333333333333333333133333333333333",
    "shift:6+8":     "3333333333333333333133333333333333",
    "shift:7+2":     "3333333333333333333133333333333333",
    "shift:7+4":     "3333333333333333333133333333333333",
    "shift:7+8":     "3333333333333333333133333333333333",
    "shift:8+2":     "3333333333333333133122222222233333",
    "shift:8+4":     "3333333333333333133122222222233333",
    "shift:8+8":     "3333333333333333133122222222233333",
    "shift:9+2":     "3333333333333333333123323323333333",
    "shift:9+4":     "3333333333333333333133313313333333",
    "shift:9+8":     "3333333333333333333133313313333333",
    "shift:10+2":    "3333333333333333333123223223233333",
    "shift:10+4":    "3333333333333333333133333333333333",
    "shift:10+8":    "3333333333333333333133333333333333",
    "shift:11+2":    "3333333333333333333123321121133333",
    "shift:11+4":    "3333333333333333333133311111133333",
    "shift:11+8":    "3333333333333333333133311111133333",
    "shift:12+2":    "3333333333333333333123321121133333",
    "shift:12+4":    "3333333333333333333133311111133333",
    "shift:12+8":    "3333333333333333333133311111133333",
    "C30_scale_o:0": "-----1---------12---------------11",
    "ref_half":      "-----3---------33-----------------",
    "scale_o:-1":    "-----2---------22---------------22",
    "scale_o:0":     "-----2---------22---------------22",
    "scale_o:nan":   "-----2---------22---------------22",
    "ws_short":      "----------------2-----------------",
}  # fmt: skip


@pytest.mark.skipif(torch.cuda.is_available(), reason="fabricated device addresses: run without a CUDA device only")
@pytest.mark.parametrize("case", CASES)
def test_entry_status(case):
    assert status_row(case) == STATUS[case]
