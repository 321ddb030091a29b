"""The grid sampler and rotate host contract without a GPU, over tables of call geometries:

* the status every grid-sampler and rotate entry returns on each row: workload shapes, extents at 0, bad ranks, grid and
  output descriptors that disagree with the input, out-of-range modes, planes at and over 2^31, null and misaligned
  pointers, bad INT8 output scales and bad rotate descriptors;
* the answers of b200_grid_sampler_supports_format, b200_rotate_supports_format and b200_dcn_supports_format for every
  (position, type, format) on representative descriptors, both plugin flavours;
* that the packed Python wrappers reject a wrong channel count or grid batch before anything reaches the library.

The entries get fabricated device addresses. An entry that accepted one of these rows would launch a kernel on them,
so the status tables run only where no CUDA device is present: there, an accepted row returns B200_ERR_LAUNCH (3) from
its first launch, and a rejected row (1 or 2) must not have counted a launch.
"""
import ctypes

import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib

no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fabricated device addresses: run without a CUDA device only")
_A = 1 << 20
BIG = (1 << 31) - 1  # the largest plane the kernels index


def _ptrs(n):
    return [_A * (i + 1) for i in range(n)]  # fabricated 256-byte-aligned device addresses, never dereferenced


def _desc(dims, dtype=0, fmt=0, scale=0.05):
    d = _lib.TensorDesc()
    d.dims.nbDims = len(dims)
    d.dims.d[: len(dims)] = dims
    d.type, d.format, d.scale = dtype, fmt, scale
    return d


def _checked(call):
    before = _lib.launch_count()
    st = call()
    if st in (1, 2):
        assert _lib.launch_count() == before, "a rejected call counted a launch"
    return st


# ---- grid sampler status -------------------------------------------------------------------------------------------------
# A row: input dims, grid dims, output dims (None: [N, C, grid spatial]), interp, padding, and a change to the call.
def _gs(idims, gdims, od=None, interp=0, pad=0, edit=None):
    return idims, gdims, od if od is not None else (*idims[:2], *gdims[2:]), interp, pad, edit


_I, _G = (2, 7, 11, 13), (2, 2, 23, 19)
_I3, _G3 = (2, 3, 4, 5, 6), (2, 3, 5, 7, 8)
GS_ROWS = {
    # workload shapes: the prev-BEV warp of the benchmark, a small call in each mode, 3-D
    "bev_warp": _gs((1, 256, 200, 200), (1, 2, 200, 200)),
    "small": _gs(_I, _G), "nearest_reflection": _gs(_I, _G, interp=1, pad=2), "bicubic_border": _gs(_I, _G, interp=2, pad=1),
    "3d": _gs(_I3, _G3), "3d_nearest": _gs(_I3, _G3, interp=1),
    # every extent at 0
    "N0": _gs((0, 7, 11, 13), (0, 2, 23, 19)), "C0": _gs((2, 0, 11, 13), _G), "Hi0": _gs((2, 7, 0, 13), _G),
    "Wi0": _gs((2, 7, 11, 0), _G), "Ho0": _gs(_I, (2, 2, 0, 19)), "Wo0": _gs(_I, (2, 2, 23, 0)),
    "od_N0": _gs(_I, _G, (0, 7, 23, 19)), "Di0": _gs((2, 3, 0, 5, 6), _G3), "Do0": _gs(_I3, (2, 3, 0, 7, 8)),
    # ranks
    "rank3": _gs((2, 7, 11), (2, 2, 23), (2, 7, 23)), "rank6": _gs((2, 7, 2, 3, 4, 5), (2, 4, 2, 3, 4, 5)),
    # grid batch and channel count
    "grid_N": _gs(_I, (3, 2, 23, 19), (2, 7, 23, 19)), "grid_ch3": _gs(_I, (2, 3, 23, 19)),
    "grid3_ch2": _gs(_I3, (2, 2, 5, 7, 8)),
    # output dims that disagree with [N, C, grid spatial]
    "od_N": _gs(_I, _G, (1, 7, 23, 19)), "od_C": _gs(_I, _G, (2, 8, 23, 19)), "od_H": _gs(_I, _G, (2, 7, 22, 19)),
    "od_W": _gs(_I, _G, (2, 7, 23, 20)), "od_D": _gs(_I3, _G3, (2, 3, 4, 7, 8)),
    # 3-D has no bicubic (and no packed layout: the "3d" rows)
    "3d_bicubic": _gs(_I3, _G3, interp=2),
    # interp / padding out of range
    "interp3": _gs(_I, _G, interp=3), "interp-1": _gs(_I, _G, interp=-1),
    "pad3": _gs(_I, _G, pad=3), "pad-1": _gs(_I, _G, pad=-1),
    # planes just below and at 2^31
    "plane_i_max": _gs((1, 4, 1, BIG), (1, 2, 8, 8)), "plane_i_over": _gs((1, 4, 2, 1 << 30), (1, 2, 8, 8)),
    "plane_o_max": _gs((1, 4, 8, 8), (1, 2, 1, BIG)), "plane_o_over": _gs((1, 4, 8, 8), (1, 2, 2, 1 << 30)),
    "plane3_i_over": _gs((1, 2, 2, 1 << 10, 1 << 20), (1, 3, 2, 2, 2)),
    "plane3_o_over": _gs((1, 2, 2, 2, 2), (1, 3, 2, 1 << 10, 1 << 20)),
    # the INT8 output scale
    "scale_o0": _gs(_I, _G, edit="scale_o0"),
    # null pointers: output, input, grid, and the three dims arrays
    **{f"null:{k}": _gs(_I, _G, edit=f"null:{k}") for k in ("out", "in", "grid", "od", "id", "gd")},
    # enqueue descriptors: grid or output rank unlike the input's
    "desc_grid_rank": _gs(_I, _G, edit="grid_rank"), "desc_out_rank": _gs(_I, _G, edit="out_rank"),
}  # fmt: skip

GS_ENTRIES = ("f32", "f16", "f16_chw2", "i8_chw4", "enq_f32", "enq_f16", "enq_chw2", "enq_i8")
_GS_ENQ = {"enq_f32": (0, 0), "enq_f16": (1, 0), "enq_chw2": (1, 1), "enq_i8": (2, 3)}


def gs_status(entry, row):
    """The status of one entry on one row, or None where the row does not apply to it."""
    idims, gdims, odims, interp, pad, edit = GS_ROWS[row]
    lib = _lib.load()
    out, inp, grid = _ptrs(3)
    nb = len(idims)
    arrays = {k: (ctypes.c_int * len(v))(*v) for k, v in (("od", odims), ("id", idims), ("gd", gdims))}
    scale_o = 0.0 if edit == "scale_o0" else 0.5
    if edit == "scale_o0" and entry not in ("i8_chw4", "enq_i8"):
        return None
    if edit in ("grid_rank", "out_rank") and entry not in _GS_ENQ:
        return None
    if edit and edit.startswith("null:"):
        what = edit[5:]
        if what in arrays:
            if entry in _GS_ENQ:
                return None
            arrays[what] = None
        else:
            out, inp, grid = (None if what == k else p for k, p in zip(("out", "in", "grid"), (out, inp, grid)))
    od, id_, gd = arrays["od"], arrays["id"], arrays["gd"]
    if entry in ("f32", "f16", "f16_chw2"):
        fn = getattr(lib, "b200_grid_sample_" + entry)
        return _checked(lambda: fn(out, inp, grid, od, id_, gd, nb, interp, pad, 0, None))
    if entry == "i8_chw4":
        return _checked(lambda: lib.b200_grid_sample_i8_chw4(out, scale_o, inp, 0.1, grid, 0.1, od, id_, gd, nb, interp,
                                                             pad, 0, None))  # fmt: skip
    dtype, fmt = _GS_ENQ[entry]
    ins = (_lib.TensorDesc * 2)(_desc(idims, dtype, fmt), _desc(gdims, dtype, fmt))
    outs = (_lib.TensorDesc * 1)(_desc(odims, dtype, fmt, scale_o))
    if edit == "grid_rank":
        ins[1].dims.nbDims = nb - 1
    if edit == "out_rank":
        outs[0].dims.nbDims = nb + 1
    inputs, outputs = (ctypes.c_void_p * 2)(inp, grid), (ctypes.c_void_p * 1)(out)
    return _checked(lambda: lib.b200_grid_sampler_enqueue(ins, outs, inputs, outputs, None, None, interp, pad, 0))


# One column per entry of GS_ENTRIES: f32 f16 f16_chw2 i8_chw4 | enq_f32 enq_f16 enq_chw2 enq_i8.
# 1 = B200_ERR_UNSUPPORTED, 2 = B200_ERR_BAD_PARAM, 3 = accepted (the first launch fails without a device), - = n/a.
GS_STATUS = {
    "bev_warp":           "33333333",
    "small":              "33333333",
    "nearest_reflection": "33333333",
    "bicubic_border":     "33333333",
    "3d":                 "33113311",
    "3d_nearest":         "33113311",
    "N0":                 "22222222",
    "C0":                 "22222222",
    "Hi0":                "22222222",
    "Wi0":                "22222222",
    "Ho0":                "22222222",
    "Wo0":                "22222222",
    "od_N0":              "22222222",
    "Di0":                "22112211",
    "Do0":                "22112211",
    "rank3":              "11112222",
    "rank6":              "11112222",
    "grid_N":             "22222222",
    "grid_ch3":           "22222222",
    "grid3_ch2":          "22112211",
    "od_N":               "22222222",
    "od_C":               "22222222",
    "od_H":               "22222222",
    "od_W":               "22222222",
    "od_D":               "22112211",
    "3d_bicubic":         "11111111",
    "interp3":            "22222222",
    "interp-1":           "22222222",
    "pad3":               "22222222",
    "pad-1":              "22222222",
    "plane_i_max":        "33333333",
    "plane_i_over":       "22222222",
    "plane_o_max":        "33333333",
    "plane_o_over":       "22222222",
    "plane3_i_over":      "22112211",
    "plane3_o_over":      "22112211",
    "scale_o0":           "---2---2",
    "null:out":           "22222222",
    "null:in":            "22222222",
    "null:grid":          "22222222",
    "null:od":            "2222----",
    "null:id":            "2222----",
    "null:gd":            "2222----",
    "desc_grid_rank":     "----2222",
    "desc_out_rank":      "----2222",
}  # fmt: skip


def gs_row(row):
    return "".join("-" if st is None else str(st) for st in (gs_status(e, row) for e in GS_ENTRIES))


@no_device
@pytest.mark.parametrize("row", list(GS_ROWS))
def test_grid_sampler_status(row):
    assert gs_row(row) == GS_STATUS[row]


# ---- rotate status -------------------------------------------------------------------------------------------------------
# A row: image dims {C, H, W}, interp, and a change to the call.
def _rot(dims, interp=0, edit=None):
    return dims, interp, edit


_R = (3, 5, 7)
ROT_ROWS = {
    # workload shapes: prev_bev of BEVFormer-base, a small call in each mode
    "bev": _rot((256, 200, 200)), "small": _rot(_R), "nearest": _rot(_R, 1),
    # every extent at 0
    "C0": _rot((0, 5, 7)), "H0": _rot((3, 0, 7)), "W0": _rot((3, 5, 0)),
    # H * W below, at half of and at 2^31 (the debug entry's output holds 2 * H * W floats)
    "HW_max": _rot((8, 1, BIG)), "HW_half": _rot((8, 1, 1 << 30)), "HW_over": _rot((8, 2, 1 << 30)),
    # interp out of range
    "interp2": _rot(_R, 2), "interp-1": _rot(_R, -1),
    # the channels-last entry wants C % 4 (fp32) / C % 8 (fp16) and 16-byte aligned buffers
    "C4": _rot((4, 5, 7)), "C6": _rot((6, 5, 7)), "C8": _rot((8, 5, 7)),
    **{f"shift:{k}+{b}": _rot((8, 5, 7), edit=f"shift:{k}+{b}") for k in ("out", "in") for b in (4, 8)},
    # the INT8 output scale
    "scale_o0": _rot(_R, edit="scale_o0"),
    # null pointers: output, input, angle, center, dims
    **{f"null:{k}": _rot(_R, edit=f"null:{k}") for k in ("out", "in", "angle", "center", "dims")},
    # enqueue descriptors
    "desc_img_rank2": _rot(_R, edit="img_rank2"), "desc_img_rank4": _rot(_R, edit="img_rank4"),
    "desc_out_rank4": _rot(_R, edit="out_rank4"), "desc_out_C": _rot(_R, edit="out_C"),
    "desc_out_W": _rot(_R, edit="out_W"), "desc_center1": _rot(_R, edit="center1"),
    "desc_angle2": _rot(_R, edit="angle2"), "desc_center_1x2": _rot(_R, edit="center_1x2"),
    "desc_angle_0d": _rot(_R, edit="angle_0d"),
}  # fmt: skip

ROT_ENTRIES = ("f32", "f16", "f16_h2", "i8", "hwc_f32", "hwc_f16", "debug", "enq_f32", "enq_f16", "enq_h2", "enq_i8")
_ROT_ENQ = {"enq_f32": (0, 0, 0), "enq_f16": (1, 0, 0), "enq_h2": (1, 1, 1), "enq_i8": (2, 3, 0)}
_ROT_DESC_EDITS = {
    "img_rank2": lambda io: setattr(io[0].dims, "nbDims", 2) or setattr(io[3].dims, "nbDims", 2),
    "img_rank4": lambda io: setattr(io[0].dims, "nbDims", 4) or setattr(io[3].dims, "nbDims", 4),
    "out_rank4": lambda io: setattr(io[3].dims, "nbDims", 4),
    "out_C": lambda io: io[3].dims.d.__setitem__(0, 4),
    "out_W": lambda io: io[3].dims.d.__setitem__(2, 6),
    "center1": lambda io: setattr(io[2].dims, "nbDims", 1) or io[2].dims.d.__setitem__(0, 1),
    "angle2": lambda io: io[1].dims.d.__setitem__(0, 2),
    "center_1x2": lambda io: setattr(io[2].dims, "nbDims", 2) or io[2].dims.d.__setitem__(0, 1) or io[2].dims.d.__setitem__(1, 2),
    "angle_0d": lambda io: setattr(io[1].dims, "nbDims", 0),
}  # fmt: skip


def rot_status(entry, row):
    """The status of one entry on one row, or None where the row does not apply to it."""
    dims, interp, edit = ROT_ROWS[row]
    lib = _lib.load()
    p = dict(zip(("out", "in", "angle", "center"), _ptrs(4)))
    cdims = (ctypes.c_int * 3)(*dims)
    scale_o = 0.0 if edit == "scale_o0" else 0.5
    if edit == "scale_o0" and entry not in ("i8", "enq_i8"):
        return None
    if edit in _ROT_DESC_EDITS and entry not in _ROT_ENQ:
        return None
    if (interp < 0 or interp > 1) and entry == "debug":
        return None
    if edit and edit.startswith("null:"):
        if edit == "null:dims":
            if entry in _ROT_ENQ:
                return None
            cdims = None
        else:
            p[edit[5:]] = None
    if edit and edit.startswith("shift:"):
        what, nbytes = edit[6:].split("+")
        p[what] += int(nbytes)
    if entry in ("f32", "f16", "f16_h2"):
        fn = getattr(lib, "b200_rotate_" + entry)
        return _checked(lambda: fn(p["out"], p["in"], p["angle"], p["center"], cdims, interp, None))
    if entry == "i8":
        return _checked(lambda: lib.b200_rotate_i8(p["out"], scale_o, p["in"], 0.1, p["angle"], p["center"], 0, cdims,
                                                   interp, None))  # fmt: skip
    if entry in ("hwc_f32", "hwc_f16"):
        dtype = int(entry == "hwc_f16")
        return _checked(lambda: lib.b200_rotate_hwc(p["out"], p["in"], p["angle"], p["center"], dtype, cdims, interp, None))
    if entry == "debug":
        return _checked(lambda: lib.b200_rotate_debug_indices(p["angle"], p["center"], cdims, p["out"], None))
    dtype, fmt, use_h2 = _ROT_ENQ[entry]
    io = (_lib.TensorDesc * 4)(_desc(dims, dtype, fmt), _desc((1,), int(dtype == 1)), _desc((2,), int(dtype == 1)),
                               _desc(dims, dtype, fmt, scale_o))  # fmt: skip
    if edit in _ROT_DESC_EDITS:
        _ROT_DESC_EDITS[edit](io)
    inputs, outputs = (ctypes.c_void_p * 3)(p["in"], p["angle"], p["center"]), (ctypes.c_void_p * 1)(p["out"])
    return _checked(lambda: lib.b200_rotate_enqueue(io, ctypes.pointer(io[3]), inputs, outputs, None, None, interp, use_h2))


# One column per entry of ROT_ENTRIES: f32 f16 f16_h2 i8 | hwc_f32 hwc_f16 | debug | enq_f32 enq_f16 enq_h2 enq_i8.
ROT_STATUS = {
    "bev":             "33333333333",
    "small":           "33331133333",
    "nearest":         "33331133333",
    "C0":              "22222222222",
    "H0":              "22222222222",
    "W0":              "22222222222",
    "HW_max":          "33333323333",
    "HW_half":         "33333323333",
    "HW_over":         "22222222222",
    "interp2":         "222222-2222",
    "interp-1":        "222222-2222",
    "C4":              "33333133333",
    "C6":              "33331133333",
    "C8":              "33333333333",
    "shift:out+4":     "33331133333",
    "shift:out+8":     "33331133333",
    "shift:in+4":      "33331133333",
    "shift:in+8":      "33331133333",
    "scale_o0":        "---2------2",
    "null:out":        "22222222222",
    "null:in":         "22222232222",
    "null:angle":      "22222222222",
    "null:center":     "22222222222",
    "null:dims":       "2222222----",
    "desc_img_rank2":  "-------2222",
    "desc_img_rank4":  "-------2222",
    "desc_out_rank4":  "-------2222",
    "desc_out_C":      "-------2222",
    "desc_out_W":      "-------2222",
    "desc_center1":    "-------2222",
    "desc_angle2":     "-------2222",
    "desc_center_1x2": "-------3333",
    "desc_angle_0d":   "-------3333",
}  # fmt: skip


def rot_row(row):
    return "".join("-" if st is None else str(st) for st in (rot_status(e, row) for e in ROT_ENTRIES))


@no_device
@pytest.mark.parametrize("row", list(ROT_ROWS))
def test_rotate_status(row):
    assert rot_row(row) == ROT_STATUS[row]


# ---- format negotiation --------------------------------------------------------------------------------------------------
# A configuration: op, the DCN groups attribute, and the descriptors (type, format, dims) TensorRT would offer, output
# last. Each is asked for every position with that position's (type, format) replaced by each of TYPES x range(4).
TYPES = (0, 1, 2, 3, 7)
F, H, I8 = 0, 1, 2
LIN, CHW2, CHW4 = 0, 1, 3
FMT_CONFIGS = {
    "gs_f32": ("gs", 1, [(F, LIN, (2, 8, 6, 6)), (F, LIN, (2, 2, 5, 5)), (F, LIN, (2, 8, 5, 5))]),
    "gs_f16": ("gs", 1, [(H, LIN, (2, 8, 6, 6)), (H, LIN, (2, 2, 5, 5)), (H, LIN, (2, 8, 5, 5))]),
    "gs_chw2": ("gs", 1, [(H, CHW2, (2, 8, 6, 6)), (H, CHW2, (2, 2, 5, 5)), (H, CHW2, (2, 8, 5, 5))]),
    "gs_i8": ("gs", 1, [(I8, CHW4, (2, 8, 6, 6)), (I8, CHW4, (2, 2, 5, 5)), (I8, CHW4, (2, 8, 5, 5))]),
    "gs3_f32": ("gs", 1, [(F, LIN, (2, 4, 3, 6, 6)), (F, LIN, (2, 3, 3, 5, 5)), (F, LIN, (2, 4, 3, 5, 5))]),
    "gs3_f16": ("gs", 1, [(H, LIN, (2, 4, 3, 6, 6)), (H, LIN, (2, 3, 3, 5, 5)), (H, LIN, (2, 4, 3, 5, 5))]),
    "rot_f32": ("rot", 1, [(F, LIN, (8, 6, 6)), (F, LIN, (1,)), (F, LIN, (2,)), (F, LIN, (8, 6, 6))]),
    "rot_f16": ("rot", 1, [(H, LIN, (8, 6, 6)), (H, LIN, (1,)), (H, LIN, (2,)), (H, LIN, (8, 6, 6))]),
    "rot_chw2": ("rot", 1, [(H, CHW2, (8, 6, 6)), (H, LIN, (1,)), (H, LIN, (2,)), (H, CHW2, (8, 6, 6))]),
    "rot_i8_f32": ("rot", 1, [(I8, CHW4, (8, 6, 6)), (F, LIN, (1,)), (F, LIN, (2,)), (I8, CHW4, (8, 6, 6))]),
    "rot_i8_f16": ("rot", 1, [(I8, CHW4, (8, 6, 6)), (H, LIN, (1,)), (H, LIN, (2,)), (I8, CHW4, (8, 6, 6))]),
    "dcn_f32": ("dcn", 1, [(F, LIN, (2, 64, 8, 8)), (F, LIN, (2, 18, 8, 8)), (F, LIN, (2, 9, 8, 8)),
                           (F, LIN, (128, 64, 3, 3)), (F, LIN, (128,)), (F, LIN, (2, 128, 8, 8))]),
    "dcn_f16": ("dcn", 1, [(H, LIN, (2, 64, 8, 8)), (H, LIN, (2, 18, 8, 8)), (H, LIN, (2, 9, 8, 8)),
                           (H, LIN, (128, 64, 3, 3)), (H, LIN, (128,)), (H, LIN, (2, 128, 8, 8))]),
    "dcn_f16_nobias": ("dcn", 1, [(H, LIN, (2, 64, 8, 8)), (H, LIN, (2, 18, 8, 8)), (H, LIN, (2, 9, 8, 8)),
                                  (H, LIN, (128, 64, 3, 3)), (H, LIN, (2, 128, 8, 8))]),
    "dcn_chw2": ("dcn", 1, [(H, CHW2, (2, 64, 8, 8)), (H, CHW2, (2, 18, 8, 8)), (H, LIN, (2, 9, 8, 8)),
                            (H, CHW2, (128, 64, 3, 3)), (H, LIN, (128,)), (H, LIN, (2, 128, 8, 8))]),
    "dcn_i8": ("dcn", 1, [(I8, CHW4, (2, 64, 8, 8)), (I8, LIN, (2, 18, 8, 8)), (I8, LIN, (2, 9, 8, 8)),
                          (I8, CHW4, (128, 64, 3, 3)), (F, LIN, (128,)), (I8, LIN, (2, 128, 8, 8))]),
    "dcn_i8_nobias": ("dcn", 1, [(I8, CHW4, (2, 64, 8, 8)), (I8, LIN, (2, 18, 8, 8)), (I8, LIN, (2, 9, 8, 8)),
                                 (I8, CHW4, (128, 64, 3, 3)), (I8, LIN, (2, 128, 8, 8))]),
    "dcn_i8_c6": ("dcn", 1, [(I8, CHW4, (2, 6, 8, 8)), (I8, LIN, (2, 18, 8, 8)), (I8, LIN, (2, 9, 8, 8)),
                             (I8, CHW4, (128, 6, 3, 3)), (F, LIN, (128,)), (I8, LIN, (2, 128, 8, 8))]),
    "dcn_i8_g64": ("dcn", 64, [(I8, CHW4, (2, 64, 8, 8)), (I8, LIN, (2, 18, 8, 8)), (I8, LIN, (2, 9, 8, 8)),
                               (I8, CHW4, (128, 1, 3, 3)), (F, LIN, (128,)), (I8, LIN, (2, 128, 8, 8))]),
}  # fmt: skip


def format_rows(name, use_h2):
    """One string per position: the answer for each (type, format) in TYPES x range(4), in that order."""
    op, groups, descs = FMT_CONFIGS[name]
    lib = _lib.load()
    nb_in = len(descs) - 1
    rows = []
    for pos in range(nb_in + 1):
        row = ""
        for t in TYPES:
            for fmt in range(4):
                io = (_lib.TensorDesc * len(descs))(*[_desc(d, dt, f) for dt, f, d in descs])
                io[pos].type, io[pos].format = t, fmt
                if op == "gs":
                    ok = lib.b200_grid_sampler_supports_format(pos, io, nb_in, 1, use_h2)
                elif op == "rot":
                    ok = lib.b200_rotate_supports_format(pos, io, nb_in, 1, use_h2)
                else:
                    ok = lib.b200_dcn_supports_format(pos, io, nb_in, 1, groups, use_h2)
                row += str(ok)
        rows.append(row)
    return rows


# The answers of the plugin shells' own rules, per configuration and flavour (0: …TRT, 1: …TRT2), one string per
# position, 20 characters each: types 0 (fp32), 1 (fp16), 2 (int8), 3 (int32), 7 (bf16) x formats 0 (linear), 1 (kCHW2),
# 2 (kHWC8), 3 (kCHW4).
FORMATS = {
    ("gs_f32", 0): ("10001000000100000000", "10000000000000000000", "10000000000000000000"),
    ("gs_f32", 1): ("10000100000100000000", "10000000000000000000", "10000000000000000000"),
    ("gs_f16", 0): ("10001000000100000000", "00001000000000000000", "00001000000000000000"),
    ("gs_f16", 1): ("10000100000100000000", "00001000000000000000", "00001000000000000000"),
    ("gs_chw2", 0): ("10001000000100000000", "00000100000000000000", "00000100000000000000"),
    ("gs_chw2", 1): ("10000100000100000000", "00000100000000000000", "00000100000000000000"),
    ("gs_i8", 0): ("10001000000100000000", "00000000000100000000", "00000000000100000000"),
    ("gs_i8", 1): ("10000100000100000000", "00000000000100000000", "00000000000100000000"),
    ("gs3_f32", 0): ("10001000000000000000", "10000000000000000000", "10000000000000000000"),
    ("gs3_f32", 1): ("10001000000000000000", "10000000000000000000", "10000000000000000000"),
    ("gs3_f16", 0): ("10001000000000000000", "00001000000000000000", "00001000000000000000"),
    ("gs3_f16", 1): ("10001000000000000000", "00001000000000000000", "00001000000000000000"),
    ("rot_f32", 0): ("10001000000100000000", "10000000000000000000", "10000000000000000000", "10000000000000000000"),
    ("rot_f32", 1): ("10000100000100000000", "10000000000000000000", "10000000000000000000", "10000000000000000000"),
    ("rot_f16", 0): ("10001000000100000000", "00001000000000000000", "00001000000000000000", "00001000000000000000"),
    ("rot_f16", 1): ("10000100000100000000", "00001000000000000000", "00001000000000000000", "00001000000000000000"),
    ("rot_chw2", 0): ("10001000000100000000", "00001000000000000000", "00001000000000000000", "00000100000000000000"),
    ("rot_chw2", 1): ("10000100000100000000", "00001000000000000000", "00001000000000000000", "00000100000000000000"),
    ("rot_i8_f32", 0): ("10001000000100000000", "10001000000000000000", "10000000000000000000", "00000000000100000000"),
    ("rot_i8_f32", 1): ("10000100000100000000", "10001000000000000000", "10000000000000000000", "00000000000100000000"),
    ("rot_i8_f16", 0): ("10001000000100000000", "10001000000000000000", "00001000000000000000", "00000000000100000000"),
    ("rot_i8_f16", 1): ("10000100000100000000", "10001000000000000000", "00001000000000000000", "00000000000100000000"),
    ("dcn_f32", 0): ("10001000000100000000", "10000000000000000000", "10000000000000000000", "10000000000000000000",
                     "10000000000000000000", "10000000000000000000"),
    ("dcn_f32", 1): ("10000100000100000000", "10000000000000000000", "10000000000000000000", "10000000000000000000",
                     "10000000000000000000", "10000000000000000000"),
    ("dcn_f16", 0): ("10001000000100000000", "00001000000000000000", "00001000000000000000", "00001000000000000000",
                     "00001000000000000000", "00001000000000000000"),
    ("dcn_f16", 1): ("10000100000100000000", "00001000000000000000", "00001000000000000000", "00001000000000000000",
                     "00001000000000000000", "00001000000000000000"),
    ("dcn_f16_nobias", 0): ("10001000000100000000", "00001000000000000000", "00001000000000000000", "00001000000000000000",
                            "00001000000000000000"),
    ("dcn_f16_nobias", 1): ("10000100000100000000", "00001000000000000000", "00001000000000000000", "00001000000000000000",
                            "00001000000000000000"),
    ("dcn_chw2", 0): ("10001000000100000000", "00000100000000000000", "00001000000000000000", "00000100000000000000",
                      "00001000000000000000", "00001000000000000000"),
    ("dcn_chw2", 1): ("10000100000100000000", "00000100000000000000", "00001000000000000000", "00000100000000000000",
                      "00001000000000000000", "00001000000000000000"),
    ("dcn_i8", 0): ("10001000000100000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                    "10001000000000000000", "00000000100000000000"),
    ("dcn_i8", 1): ("10000100000100000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                    "10001000000000000000", "00000000100000000000"),
    ("dcn_i8_nobias", 0): ("10001000000100000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                           "00000000100000000000"),
    ("dcn_i8_nobias", 1): ("10000100000100000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                           "00000000100000000000"),
    ("dcn_i8_c6", 0): ("10001000000000000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                       "10001000000000000000", "00000000100000000000"),
    ("dcn_i8_c6", 1): ("10000100000000000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                       "10001000000000000000", "00000000100000000000"),
    ("dcn_i8_g64", 0): ("10001000000000000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                        "10001000000000000000", "00000000100000000000"),
    ("dcn_i8_g64", 1): ("10000100000000000000", "00000000100000000000", "00000000100000000000", "00000000000100000000",
                        "10001000000000000000", "00000000100000000000"),
}  # fmt: skip


@pytest.mark.parametrize("use_h2", [0, 1])
@pytest.mark.parametrize("name", list(FMT_CONFIGS))
def test_supports_format(name, use_h2):
    assert tuple(format_rows(name, use_h2)) == FORMATS[name, use_h2]


# ---- Python wrappers of the packed layouts ---------------------------------------------------------------------------------
def _no_library(monkeypatch):
    def refuse(*_a, **_k):
        raise AssertionError("the call reached the library")

    monkeypatch.setattr(_lib, "call", refuse)


def test_packed_grid_sampler_wrappers_check_shapes_first(monkeypatch):
    _no_library(monkeypatch)
    x2, g2 = torch.zeros(2, 4, 6, 6, 2, dtype=torch.float16), torch.zeros(2, 1, 5, 5, 2, dtype=torch.float16)
    x4, g4 = torch.zeros(2, 2, 6, 6, 4, dtype=torch.int8), torch.zeros(2, 1, 5, 5, 4, dtype=torch.int8)
    chw2 = lambda x, g, c: bt.grid_sampler_chw2(x, g, c, "bilinear", "zeros", False)  # noqa: E731
    int8 = lambda x, g, c: bt.grid_sampler_int8(x, 0.1, g, 0.1, 0.5, c, "bilinear", "zeros", False)  # noqa: E731
    for call, x, g, good, bad in ((chw2, x2, g2, 8, (9, 6, 100)), (int8, x4, g4, 8, (9, 4, 100))):
        for c in bad:  # ceil(c / width) != the packet count: the kernel would read and write past both tensors
            with pytest.raises(ValueError, match="input must be"):
                call(x, g, c)
        with pytest.raises(ValueError, match="grid must be"):  # the grid's batch differs from the input's
            call(x, g[:1], good)
        with pytest.raises(ValueError, match="grid must be"):
            call(x, torch.cat([g, g]), good)
        with pytest.raises(RuntimeError, match="CUDA"):  # shapes fine: the CPU tensors are refused next
            call(x, g, good)
        with pytest.raises(RuntimeError, match="CUDA"):
            call(x, g, good - 1)  # 7 channels still fill the last packet's slot


def test_packed_rotate_wrappers_check_shapes_first(monkeypatch):
    _no_library(monkeypatch)
    angle, center = torch.tensor([3.0]), torch.tensor([2.0, 2.0])
    x2, x4 = torch.zeros(4, 5, 5, 2, dtype=torch.float16), torch.zeros(2, 5, 5, 4, dtype=torch.int8)
    chw2 = lambda x, c: bt.rotate_chw2(x, c, angle, center)  # noqa: E731
    int8 = lambda x, c: bt.rotate_int8(x, 0.1, c, angle, center, 0.5)  # noqa: E731
    for call, x, good, bad in ((chw2, x2, 8, (9, 6, 0, 100)), (int8, x4, 8, (9, 4, 0, 100))):
        for c in bad:
            with pytest.raises(ValueError, match="img must be"):
                call(x, c)
        with pytest.raises(ValueError, match="img must be"):
            call(x[None], good)
        with pytest.raises(RuntimeError, match="CUDA"):
            call(x, good)
