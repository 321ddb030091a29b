"""The DCNv2 host contract without a GPU, over one table of layer geometries:

* the exact bytes every DCN workspace query returns (these queries never touch a device, so they run everywhere);
* the status every DCN launcher returns on each geometry and on null, misaligned or out-of-range arguments.

The launchers get fabricated device addresses. A launcher that accepted one of these rows would launch a kernel on
them, so the status table runs only where no CUDA device is present: there, an accepted row returns
B200_ERR_LAUNCH (3) from its first launch, and a rejected row (1 or 2) must not have counted a launch.
"""
import ctypes

import pytest
import torch

from bevformer_tensorrt_b200 import _lib

# The C ABI's argument order: batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h,
# pad_w, pad_h, dilation_w, dilation_h, group, deformable_group.
GEO = {
    "base": (6, 256, 58, 100, 256, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "base_co128": (6, 256, 58, 100, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "base_co512_s2": (6, 512, 58, 100, 512, 3, 3, 2, 2, 1, 1, 1, 1, 1, 1),
    "small": (2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "groups2_dg2": (2, 16, 13, 17, 12, 3, 3, 1, 1, 1, 1, 1, 1, 2, 2),
    "groups4_dg2": (2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 4, 2),
    "asym": (2, 64, 31, 45, 128, 5, 3, 2, 1, 2, 0, 1, 2, 1, 1),
    "k1x9": (1, 64, 16, 40, 128, 9, 1, 1, 1, 4, 0, 1, 1, 1, 1),
    "k7x7": (1, 64, 24, 24, 128, 7, 7, 1, 1, 3, 3, 1, 1, 1, 1),
    "k8x9": (1, 32, 24, 24, 64, 9, 8, 1, 1, 4, 4, 1, 1, 1, 1),
    "k9x9": (1, 32, 24, 24, 64, 9, 9, 1, 1, 4, 4, 1, 1, 1, 1),
    "k13x13": (1, 16, 30, 30, 32, 13, 13, 1, 1, 6, 6, 1, 1, 1, 1),
    "over_2g": (1, 4096, 300, 300, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),  # channels * taps * Ho * Wo >= 2^31
    # edge rows
    "batch0": (0, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "channels0": (2, 0, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "height0": (2, 64, 0, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "width0": (2, 64, 20, 0, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "co0": (2, 64, 20, 24, 0, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "kernel0": (2, 64, 20, 24, 128, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1),
    "stride0": (2, 64, 20, 24, 128, 3, 3, 1, 0, 1, 1, 1, 1, 1, 1),
    "dilation0": (2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 0, 1, 1, 1),
    "pad_neg": (2, 64, 20, 24, 128, 3, 3, 1, 1, -1, 1, 1, 1, 1, 1),
    "no_output": (2, 64, 2, 24, 128, 3, 3, 1, 1, 1, -1, 1, 1, 1, 1),  # Ho = 0
    "trunc": (1, 64, 2, 2, 128, 3, 3, 2, 2, 0, 0, 1, 1, 1, 1),  # numerator -1: truncation gives Ho = Wo = 1
    "group0": (2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 0, 1),
    "dg0": (2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 0),
    "c_mod_group": (2, 18, 13, 17, 12, 3, 3, 1, 1, 1, 1, 1, 1, 4, 1),
    "co_mod_group": (2, 16, 13, 17, 10, 3, 3, 1, 1, 1, 1, 1, 1, 4, 1),
    "c_mod_dg": (2, 16, 13, 17, 12, 3, 3, 1, 1, 1, 1, 1, 1, 1, 3),
    "c_mod4": (2, 18, 13, 17, 12, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1),  # kCHW4 packs 4 channels
}


def _extent(size, k, s, p, d):
    """The launchers' output extent: C's truncating division."""
    n = size + 2 * p - (d * (k - 1) + 1)
    return (n // s if n >= 0 else -(-n // s)) + 1 if s > 0 else 0


def _enqueue_descs(geo, dtype, fmt):
    """Descriptors of the layer `geo` as TensorRT would pass them to b200_dcn_enqueue[_workspace_size], with the
    attribute arrays in ONNX order (h, w)."""
    n, c, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, g, dg = geo
    ho, wo = _extent(h, kh, sh, ph, dh), _extent(w, kw, sw, pw, dw)
    shapes = [(n, c, h, w), (n, dg * 2 * kh * kw, ho, wo), (n, dg * kh * kw, ho, wo), (co, c // g if g else c, kh, kw),
              (co,)]  # fmt: skip
    ins = (_lib.TensorDesc * 5)()
    for d, s in zip(ins, shapes):
        d.dims.nbDims = len(s)
        d.dims.d[: len(s)] = s
        d.type, d.format, d.scale = dtype, fmt, 0.05
    out = (_lib.TensorDesc * 1)()
    out[0].dims.nbDims = 4
    out[0].dims.d[:4] = (n, co, ho, wo)
    out[0].type, out[0].format, out[0].scale = dtype, fmt, 0.05
    arr = lambda a, b: (ctypes.c_int32 * 2)(a, b)  # noqa: E731
    return ins, out, arr(sh, sw), arr(ph, pw), arr(dh, dw)


# ---- workspace queries ---------------------------------------------------------------------------------------------------
# b200_dcn_enqueue_workspace_size flavours: (type, format) of the input descriptor
ENQ = {"enq_f32": (0, 0), "enq_f16": (1, 0), "enq_f16_chw2": (1, 1), "enq_i8": (2, 3)}
WS_COLUMNS = ("f32", "f16", "bf16", "i8", "f16_chw2", "bw_f32", "bw_f16", "bw_bf16", *ENQ)


def workspace_row(geo):
    lib = _lib.load()
    fwd = geo[:4] + geo[5:13]  # b200_dcn_workspace_size has no channels_out, group or deformable_group
    row = [lib.b200_dcn_workspace_size(d, *fwd) for d in (0, 1, 7)]
    row += [lib.b200_dcn_i8_workspace_size(*geo), lib.b200_dcn_f16_chw2_workspace_size(*geo)]
    row += [lib.b200_dcn_backward_workspace_size(d, *geo) for d in (0, 1, 7)]
    for dtype, fmt in ENQ.values():
        ins, _, stride, padding, dilation = _enqueue_descs(geo, dtype, fmt)
        row.append(lib.b200_dcn_enqueue_workspace_size(ins, stride, padding, dilation, geo[13], geo[14]))
    return dict(zip(WS_COLUMNS, row))


WS = {
    "base": (256, 20178944, 256, 38694656, 40429056, 41424896, 77060096, 77060096, 256, 20178944, 40429056, 38694656),
    "base_co128": (256, 20178944, 256, 29195776, 39839232, 41424896, 77060096, 77060096, 256, 20178944, 39839232, 29195776),
    "base_co512_s2": (256, 40355840, 256, 49733632, 81022976, 40485376, 111755776, 111755776, 256, 40355840, 81022976, 49733632),
    "small": (256, 714752, 256, 714752, 1019648, 6377472, 6623232, 6623232, 256, 714752, 1019648, 714752),
    "groups2_dg2": (256, 163840, 256, 163840, 211968, 218624, 247040, 247040, 256, 163840, 211968, 163840),
    "groups4_dg2": (256, 714752, 256, 714752, 943616, 2838528, 3084288, 3084288, 256, 714752, 943616, 714752),
    "asym": (256, 1342208, 256, 1342208, 2019840, 16984320, 17698560, 17698560, 256, 1342208, 2019840, 1342208),
    "k1x9": (256, 673792, 256, 673792, 926208, 4055040, 4218880, 4218880, 256, 673792, 926208, 673792),
    "k7x7": (256, 3287040, 256, 3287040, 4276480, 32150272, 32297728, 32297728, 256, 3287040, 4276480, 3287040),
    "k8x9": (256, 2398208, 256, 2398208, 2902784, 22487040, 22560768, 22560768, 256, 2398208, 2902784, 2398208),
    "k9x9": (256, 2693120, 256, 2693120, 3248384, 0, 0, 0, 256, 2693120, 3248384, 2693120),
    "k13x13": (256, 2799872, 256, 2799872, 3610368, 0, 0, 0, 256, 2799872, 3610368, 2799872),
    "over_2g": (256, 775030784, 256, 775030784, 1524988160, 0, 0, 0, 256, 775030784, 1524988160, 775030784),
    "batch0": (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "channels0": (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "height0": (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "width0": (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "co0": (256, 714752, 256, 0, 0, 0, 0, 0, 256, 714752, 0, 0),
    "kernel0": (256, 124928, 256, 399616, 247808, 0, 0, 0, 256, 124928, 247808, 399616),
    "stride0": (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "dilation0": (256, 714752, 256, 714752, 1022720, 0, 0, 0, 256, 714752, 1022720, 714752),
    "pad_neg": (256, 714752, 256, 714752, 1014016, 0, 0, 0, 256, 714752, 1014016, 714752),
    "no_output": (0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
    "trunc": (256, 592384, 256, 592384, 740608, 296704, 297728, 297728, 256, 592384, 740608, 592384),
    "group0": (256, 714752, 256, 0, 0, 0, 0, 0, 256, 714752, 0, 0),
    "dg0": (256, 714752, 256, 0, 0, 0, 0, 0, 256, 714752, 0, 0),
    "c_mod_group": (256, 184064, 256, 184064, 217344, 0, 0, 0, 256, 184064, 217344, 184064),
    "co_mod_group": (256, 163840, 256, 163840, 195072, 0, 0, 0, 256, 163840, 195072, 163840),
    "c_mod_dg": (256, 163840, 256, 163840, 229632, 0, 0, 0, 256, 163840, 229632, 163840),
    "c_mod4": (256, 184064, 256, 184064, 220416, 492032, 524032, 524032, 256, 184064, 220416, 184064),
}  # fmt: skip


@pytest.mark.parametrize("name", list(GEO))
def test_workspace_bytes(name):
    assert workspace_row(GEO[name]) == dict(zip(WS_COLUMNS, WS[name]))


# ---- launcher status -----------------------------------------------------------------------------------------------------
_A = 1 << 20
_WS = _A * 64  # 256-byte aligned


def _ptrs():
    return [_A * (i + 1) for i in range(10)]  # fabricated 256-byte-aligned device addresses, never dereferenced


def _call(entry, geo, ptrs, ws, flags=0, scale_o=0.5):
    """Calls the DCN launcher `entry` on `geo`. Forward pointer slots: input 0, weight 1, bias 2, offset 3, mask 4,
    output 5. Backward: input 0, weight 1, offset 2, mask 3, grad_output 4, grad_input / weight / bias / offset / mask
    5-9. enq_*: b200_dcn_enqueue with 5 inputs (slots 0-4 in the plugin's order x, offset, mask, weight, bias)."""
    lib = _lib.load()
    if entry in ("f32", "f16", "bf16", "f16_chw2"):
        return getattr(lib, "b200_dcn_" + entry)(*ptrs[:6], ws, *geo, 1, None, None)
    if entry == "f16_ex":
        return lib.b200_dcn_f16_ex(*ptrs[:6], ws, *geo, flags, None)
    if entry == "i8":
        p = ptrs
        return lib.b200_dcn_i8(p[0], 0.1, p[1], 0.1, p[2], 0, p[3], 0.1, p[4], 0.1, p[5], scale_o, ws, *geo, 1, None, None)
    if entry == "pack":
        return lib.b200_dcn_pack_weights_f16(ptrs[1], ptrs[6], geo[4], geo[1], geo[6], geo[5], None)
    if entry == "bw_f16":
        return lib.b200_dcn_backward_f16(*ptrs[:10], ws, *geo, flags, None)
    if entry in ("bw_f32", "bw_bf16"):
        return getattr(lib, "b200_dcn_backward_" + entry[3:])(*ptrs[:10], ws, *geo, None)
    ins, out, stride, padding, dilation = _enqueue_descs(geo, *ENQ[entry])
    inputs, outputs = (ctypes.c_void_p * 5)(*ptrs[:5]), (ctypes.c_void_p * 1)(ptrs[5])
    return lib.b200_dcn_enqueue(ins, out, inputs, outputs, ws, None, 5, stride, padding, dilation, geo[13], geo[14])


ENTRIES = ("f32", "f16", "bf16", "f16_chw2", "f16_ex", "i8", "pack", "bw_f32", "bw_f16", "bw_bf16", *ENQ)


def _case(case):
    """(geometry, pointers, workspace, keyword arguments) of a status row: a GEO name, or a change to the "small" layer."""
    ptrs, ws, kw = _ptrs(), _WS, {}
    if case in GEO:
        return GEO[case], ptrs, ws, kw
    what, _, arg = case.partition(":")
    if what == "null":
        ptrs[int(arg)] = None
    elif what == "shift":  # "shift:<slot>+<bytes>"
        slot, nbytes = map(int, arg.split("+"))
        ptrs[slot] += nbytes
    elif what == "ws_null":
        ws = None
    elif what == "ws_shift":
        ws += int(arg)
    elif what == "flags":
        kw["flags"] = int(arg)
    elif what == "scale_o":
        kw["scale_o"] = float(arg)
    return GEO["small"], ptrs, ws, kw


def status(entry, case):
    geo, ptrs, ws, kw = _case(case)
    before = _lib.launch_count()
    st = _call(entry, geo, ptrs, ws, **kw)
    if st in (1, 2):
        assert _lib.launch_count() == before, "a rejected call counted a launch"
    return st


POINTER_CASES = ([f"null:{i}" for i in range(10)] + [f"shift:{i}+{b}" for i in range(10) for b in (1, 2, 8)] +
                 ["ws_null", "ws_shift:2", "ws_shift:128"])  # fmt: skip
EXTRA_CASES = {"f16_ex": ["flags:1", "flags:3"], "i8": ["scale_o:0", "scale_o:nan", "scale_o:-1"],
               "bw_f16": ["flags:1", "flags:3", "flags:4"]}  # fmt: skip
CASES = list(GEO) + POINTER_CASES + sorted({c for cs in EXTRA_CASES.values() for c in cs})


def status_row(case):
    """One character per entry of ENTRIES: its status, or "-" where the case does not apply to it."""
    extra = case in CASES[len(GEO) + len(POINTER_CASES):]
    return "".join("-" if extra and case not in EXTRA_CASES.get(e, ()) else str(status(e, case)) for e in ENTRIES)


# One column per entry of ENTRIES: f32 f16 bf16 f16_chw2 f16_ex i8 pack bw_f32 bw_f16 bw_bf16 enq_f32 enq_f16
# enq_f16_chw2 enq_i8. 1 = B200_ERR_UNSUPPORTED, 2 = B200_ERR_BAD_PARAM, 3 = accepted (the first launch fails without a
# device).
STATUS = {
    "base":          "33333333333333",
    "base_co128":    "33333333333333",
    "base_co512_s2": "33333333333333",
    "small":         "33333333333333",
    "groups2_dg2":   "33331313333333",
    "groups4_dg2":   "33331333333333",
    "asym":          "33331313333333",
    "k1x9":          "33333333333333",
    "k7x7":          "33331313333333",
    "k8x9":          "33331313333333",
    "k9x9":          "33331311113333",
    "k13x13":        "11131311111133",
    "over_2g":       "22233332222233",
    "batch0":        "22222232222222",
    "channels0":     "22222222222222",
    "height0":       "22222232222222",
    "width0":        "22222232222222",
    "co0":           "22222222222222",
    "kernel0":       "22222222222222",
    "stride0":       "22222232222222",
    "dilation0":     "22222232222222",
    "pad_neg":       "33333332222222",
    "no_output":     "22222232222222",
    "trunc":         "33333333332222",
    "group0":        "22222232222222",
    "dg0":           "22222232222222",
    "c_mod_group":   "11111112222222",
    "co_mod_group":  "11111112221111",
    "c_mod_dg":      "11111112221111",
    "c_mod4":        "33331113333331",
    "null:0":        "22222232222222",
    "null:1":        "22222222222222",
    "null:2":        "33333332222222",
    "null:3":        "22222232222222",
    "null:4":        "22222232223333",
    "null:5":        "22222233332222",
    "null:6":        "33333323333333",
    "null:7":        "33333333333333",
    "null:8":        "33333333333333",
    "null:9":        "33333333333333",
    "shift:0+1":     "33331132223331",
    "shift:0+2":     "33331132333331",
    "shift:0+8":     "33331333333333",
    "shift:1+1":     "33331132223333",
    "shift:1+2":     "33331132333333",
    "shift:1+8":     "33331333333333",
    "shift:2+1":     "33333332223333",
    "shift:2+2":     "33333332333333",
    "shift:2+8":     "33333333333333",
    "shift:3+1":     "33333332223331",
    "shift:3+2":     "33333332333331",
    "shift:3+8":     "33333333333333",
    "shift:4+1":     "33333332223333",
    "shift:4+2":     "33333332333333",
    "shift:4+8":     "33333333333333",
    "shift:5+1":     "33333332223333",
    "shift:5+2":     "33333332333333",
    "shift:5+8":     "33333333333333",
    "shift:6+1":     "33333332223333",
    "shift:6+2":     "33333332333333",
    "shift:6+8":     "33333333333333",
    "shift:7+1":     "33333332223333",
    "shift:7+2":     "33333332333333",
    "shift:7+8":     "33333333333333",
    "shift:8+1":     "33333332223333",
    "shift:8+2":     "33333332333333",
    "shift:8+8":     "33333333333333",
    "shift:9+1":     "33333332223333",
    "shift:9+2":     "33333332333333",
    "shift:9+8":     "33333333333333",
    "ws_null":       "33322232223322",
    "ws_shift:2":    "33311132223311",
    "ws_shift:128":  "33311132223311",
    "flags:1":       "----3---3-----",
    "flags:3":       "----3---3-----",
    "flags:4":       "--------2-----",
    "scale_o:-1":    "-----2--------",
    "scale_o:0":     "-----2--------",
    "scale_o:nan":   "-----2--------",
}  # fmt: skip


@pytest.mark.skipif(torch.cuda.is_available(), reason="fabricated device addresses: run without a CUDA device only")
@pytest.mark.parametrize("case", CASES)
def test_launcher_status(case):
    want = STATUS[case]
    # b200_dcn_f16_ex returns BAD_PARAM (2) for a non-positive group or deformable-group count, like every other
    # launcher. Library versions 0.1.0 and older returned UNSUPPORTED (1).
    if case in ("group0", "dg0") and b" 0.1.0 " in _lib.load().b200_bev_ops_version():
        i = ENTRIES.index("f16_ex")
        want = want[:i] + "1" + want[i + 1 :]
    assert status_row(case) == want
