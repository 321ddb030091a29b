"""oracle/f64.py — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Float64 references of multi-scale deformable attention and DCNv2, forward and backward, and of rotate's sampling step,
written from the definition of each op in plain torch. Every output and gradient element ``e`` comes with what a per-element rounding bound needs:

* ``r``    its value;
* ``mag``  the sum of |terms| that make up ``r`` (the same computation on magnitudes where the op is monotone; written out
           where a gradient holds differences, so that ``|v01| - |v00|`` becomes ``|v01| + |v00|``);
* ``n``    the length of the longest chain of sums behind ``r`` (inner sum plus outer sum for a sum of sums): the
           classic bound ``n * u * mag`` on a float sum holds for any summation order, atomics included;
  For MSDA every chain also carries the softmax: a weight ``a_k = e_k / sum_j e_j`` with ``e_k = exp(l_k - max l)``
           is within ``(NP + (max l - min l) + 6) u`` of its value, relative (the rounding of the exponent's argument,
           at most ``max l - min l`` units; expf's 2 ulp; the NP-term denominator; the division), so that count
           joins n: the forward's n is 4 (corners) + NP (points) + that softmax count.
* ``lmag`` / ``lcnt`` where a path rounds an intermediate to FP16 / BF16 (see the functions): the magnitude of the
           rounded values times the number of roundings each goes through, and the count of those roundings weighted
           like their values, for the subnormal range, where a rounding errs by half the smallest subnormal
           absolutely rather than relatively.
* ``pmag`` (MSDA only) the sensitivity of ``r`` to the fp32 rounding of the sampling positions, in units of 2^-24: the
           kernel forms ``x = ref * W + off - 0.5`` in fp32, which moves ``x`` by at most
           ``2^-24 * (|ref * W| + |ref * W + off| + |x|) <= 3 * 2^-24 * (|ref * W| + |off| + 1/2)``, and a bilinear weight
           moves by at most the position error per axis. DCN needs no such term: its positions are the fp32 sums the
           kernel forms (``base + offset``), taken exactly into float64.

The inputs are the tensors the kernel reads (rounded to the call's dtype, then widened). Where the bilinear derivative
jumps (a position on an integer), the references take the cell the kernel takes: MSDA from the index records of the
FP32 oracle (``oracle.msda.msda_f32(..., return_index=True)``), which are the kernel's bit for bit; DCN from ``floor`` of
the fp32 position, with mmcv's range rule (a sample at exactly -1 or at H / W is outside and has no gradient).
"""
import numpy as np
import torch

from .msda import msda_f32

F64 = torch.float64
_TAPS = ((0, 0), (0, 1), (1, 0), (1, 1))  # corner t = (dy, dx): top-left, top-right, bottom-left, bottom-right


def _entry(r, mag, n, pmag=None, lmag=None, lcnt=None):
    z = torch.zeros_like(r)
    n = torch.as_tensor(n, dtype=F64, device=r.device).expand_as(r)
    return {"r": r, "mag": mag, "n": n, "pmag": z if pmag is None else pmag, "lmag": z if lmag is None else lmag,
            "lcnt": z if lcnt is None else lcnt}


def msda_index(value, shapes, ref, off, logits):
    """The FP32 oracle's sampling-index records for these inputs (only the positions matter: value is not read)."""
    B, S, M, C = value.shape
    f32 = lambda t: t.detach().float().cpu().numpy()  # noqa: E731
    dummy_v = np.zeros((B, S, M, 1), np.float32)
    _, idx = msda_f32(dummy_v, shapes.cpu().numpy(), f32(ref), f32(off), f32(logits), return_index=True)
    return idx


def msda_f64(value, shapes, ref, off, logits, grad_out=None, index=None, device="cpu", budget=1 << 21):
    """value [B,S,M,C], shapes int [L,2] (h, w), ref [B,Q,1,2G], off [B,Q,M,L*P*2] in pixels, logits [B,Q,M,L*P]
    pre-softmax, grad_out [B,Q,M,C] or None. Returns {"out": entry} and, with grad_out, "grad_value", "grad_ref",
    "grad_off", "grad_logits" entries in the inputs' shapes (float64 on ``device``). ``budget`` bounds the elements
    of one gathered [B, q, M, L*P, C] block (queries are processed in chunks)."""
    dev = torch.device(device)
    B, S, M, C = value.shape
    L = shapes.shape[0]
    Q, NP, G = off.shape[1], logits.shape[-1], ref.shape[-1] // 2
    P = NP // L
    if index is None:
        index = msda_index(value, shapes, ref, off, logits)
    hw = shapes.cpu().long().tolist()
    lvl = torch.arange(NP) // P
    Hk = torch.tensor([hw[l][0] for l in lvl.tolist()], dtype=F64, device=dev)
    Wk = torch.tensor([hw[l][1] for l in lvl.tolist()], dtype=F64, device=dev)
    starts = np.cumsum([0] + [h * w for h, w in hw])[:-1]
    startk = torch.tensor(starts[lvl.numpy()], dtype=torch.long, device=dev)
    Hi, Wi = Hk.long(), Wk.long()
    gk = (torch.arange(NP) % P % G).to(dev)

    v64 = value.detach().to(dev, F64)
    want_grad = grad_out is not None
    out = {k: torch.zeros(B, Q, M, C, dtype=F64, device=dev) for k in ("r", "mag", "pmag")}
    if want_grad:
        gv = {k: torch.zeros(B * S * M, C, dtype=F64, device=dev) for k in ("r", "mag", "pmag")}
        gv_count = torch.zeros(B * S * M, dtype=F64, device=dev)
        goff = {k: torch.zeros(B, Q, M, NP, 2, dtype=F64, device=dev) for k in ("r", "mag", "pmag")}
        glog = {k: torch.zeros(B, Q, M, NP, dtype=F64, device=dev) for k in ("r", "mag", "pmag")}
        gref = {k: torch.zeros(B, Q, G, 2, dtype=F64, device=dev) for k in ("r", "mag", "pmag")}
    soft = torch.zeros(B, Q, M, dtype=F64, device=dev)  # the softmax's share of every chain (module docstring)
    chunk = max(1, budget // max(1, B * M * NP * C))
    bidx = torch.arange(B, device=dev).view(B, 1, 1, 1)
    midx = torch.arange(M, device=dev).view(1, 1, M, 1)
    for q0 in range(0, Q, chunk):
        q1 = min(Q, q0 + chunk)
        r = ref[:, q0:q1].detach().to(dev, F64).reshape(B, q1 - q0, G, 2)
        o = off[:, q0:q1].detach().to(dev, F64).reshape(B, q1 - q0, M, NP, 2)
        lg = logits[:, q0:q1].detach().to(dev, F64)
        rx, ry = r[:, :, gk, 0].unsqueeze(2), r[:, :, gk, 1].unsqueeze(2)  # [B, q, 1, NP]
        x = rx * Wk + o[..., 0] - 0.5
        y = ry * Hk + o[..., 1] - 0.5
        rec = {k: torch.from_numpy(np.ascontiguousarray(index[k][:, q0:q1])).to(dev).long()
               for k in ("in_range", "h_low", "w_low", "tap_mask")}  # fmt: skip
        ok, hl, wl, tm = rec["in_range"] != 0, rec["h_low"], rec["w_low"], rec["tap_mask"]
        lh, lw = y - hl, x - wl
        hh, hw_ = 1 - lh, 1 - lw
        valid = torch.stack([ok & (((tm >> t) & 1) != 0) for t in range(4)])  # [4, B, q, M, NP]
        wts = torch.stack([hh * hw_, hh * lw, lh * hw_, lh * lw]) * valid
        pix = torch.stack([startk + (hl + dy).clamp(min=0).minimum(Hi - 1) * Wi + (wl + dx).clamp(min=0).minimum(Wi - 1)
                           for dy, dx in _TAPS])  # fmt: skip
        vt = torch.stack([v64[bidx, pix[t], midx] for t in range(4)]) * valid.unsqueeze(-1)  # [4, B, q, M, NP, C]
        va = vt.abs()
        att = lg.softmax(-1)
        soft[:, q0:q1] = NP + (lg.amax(-1) - lg.amin(-1)) + 6
        Pk = 3 * ((rx * Wk).abs() + o[..., 0].abs() + (ry * Hk).abs() + o[..., 1].abs() + 1)  # [B, q, M, NP]
        s = (wts.unsqueeze(-1) * vt).sum(0)  # [B, q, M, NP, C]
        sa = (wts.unsqueeze(-1) * va).sum(0)
        V = va.sum(0)
        a = att.unsqueeze(-1)
        out["r"][:, q0:q1] = (a * s).sum(3)
        out["mag"][:, q0:q1] = (a * sa).sum(3)
        out["pmag"][:, q0:q1] = (a * Pk.unsqueeze(-1) * V).sum(3)
        if not want_grad:
            continue
        go = grad_out[:, q0:q1].detach().to(dev, F64)  # [B, q, M, C]
        ga = go.abs().unsqueeze(3)
        go3 = go.unsqueeze(3)
        d, D, PD = (go3 * s).sum(-1), (ga * sa).sum(-1), (ga * V).sum(-1) * Pk
        glog["r"][:, q0:q1] = att * (d - (att * d).sum(-1, keepdim=True))
        glog["mag"][:, q0:q1] = att * (D + (att * D).sum(-1, keepdim=True))
        glog["pmag"][:, q0:q1] = att * (PD + (att * PD).sum(-1, keepdim=True))
        hh_, lh_, hw2, lw_ = (t.unsqueeze(-1) for t in (hh, lh, hw_, lw))
        dx_r = (go3 * (hh_ * (vt[1] - vt[0]) + lh_ * (vt[3] - vt[2]))).sum(-1) * att
        dy_r = (go3 * (hw2 * (vt[2] - vt[0]) + lw_ * (vt[3] - vt[1]))).sum(-1) * att
        dx_m = (ga * (hh_ * (va[1] + va[0]) + lh_ * (va[3] + va[2]))).sum(-1) * att
        dy_m = (ga * (hw2 * (va[2] + va[0]) + lw_ * (va[3] + va[1]))).sum(-1) * att
        dp = att * PD  # both axes: the derivative of one axis moves with the other axis' position
        goff["r"][:, q0:q1] = torch.stack([dx_r, dy_r], -1)
        goff["mag"][:, q0:q1] = torch.stack([dx_m, dy_m], -1)
        goff["pmag"][:, q0:q1] = torch.stack([dp, dp], -1)
        onehot = (gk.view(NP, 1) == torch.arange(G, device=dev).view(1, G)).to(F64)  # [NP, G]
        for key, (ax, ay) in (("r", (dx_r, dy_r)), ("mag", (dx_m, dy_m)), ("pmag", (dp, dp))):
            gref[key][:, q0:q1, :, 0] = torch.einsum("bqmk,kg->bqg", ax * Wk, onehot)
            gref[key][:, q0:q1, :, 1] = torch.einsum("bqmk,kg->bqg", ay * Hk, onehot)
        flat = ((bidx * S + pix) * M + midx).reshape(-1)  # [4 * B * q * M * NP]
        aw = (att * wts).unsqueeze(-1)  # [4, B, q, M, NP, 1]
        gv["r"].index_add_(0, flat, (aw * go3).reshape(-1, C))
        gv["mag"].index_add_(0, flat, (aw * ga).reshape(-1, C))
        gv["pmag"].index_add_(0, flat, ((att * Pk * valid).unsqueeze(-1) * ga).reshape(-1, C))
        gv_count.index_add_(0, flat, valid.reshape(-1).to(F64))
    sk = soft.unsqueeze(-1)  # [B, Q, M, 1]
    res = {"out": _entry(out["r"], out["mag"], 4 + NP + sk, out["pmag"])}
    if want_grad:
        res["grad_value"] = _entry(gv["r"].view(B, S, M, C), gv["mag"].view(B, S, M, C),
                                   (gv_count + 4).view(B, S, M, 1) + soft.max(), gv["pmag"].view(B, S, M, C))
        res["grad_off"] = _entry(*(goff[k].reshape(B, Q, M, NP * 2) for k in ("r", "mag")), 4 * C + 4 + sk,
                                 goff["pmag"].reshape(B, Q, M, NP * 2))  # fmt: skip
        res["grad_logits"] = _entry(glog["r"], glog["mag"], 4 * C + NP + 4 + sk, glog["pmag"])
        res["grad_ref"] = _entry(*(gref[k].reshape(B, Q, 1, 2 * G) for k in ("r", "mag")),
                                 4 * C + 4 + M * NP + soft.amax(2).view(B, Q, 1, 1), gref["pmag"].reshape(B, Q, 1, 2 * G))
    return res


def msda_sca_f64(value, shapes, ref, off, logits, mask, grad_slots=None, shared=False, device="cpu"):
    """The fused spatial-cross-attention forms: slots [Q, M*C] = sum_b mask[b, q] * MSDA(value[b], ref[b], ...)[b, q].
    ``shared``: offsets / logits are one copy [1, Q, M, .] for every camera, and their gradients are summed over the
    cameras. Backward: grad_out of camera b is mask[b, q] * grad_slots[q]. Same entries as ``msda_f64``.

    ``lmag`` / ``lcnt`` describe the fallback these forms take outside the fused kernel's envelope, which rounds to the
    value dtype (functions/multi_scale_deformable_attn.py:462-471, 503-507): forward, each camera's output once
    (``|out_b|`` is at most ``|r_b|`` plus its fp32 error); backward, each grad_out element once, which moves every
    gradient by at most the rounding times its ``mag`` (the gradients are linear in grad_out), and for the shared form
    each camera's offset and logit gradient once more before the camera sum (at most ``mag_b`` each, with a 2^-6
    allowance for their own error). ``lcnt`` counts the same roundings with grad_out's magnitude taken as 1."""
    dev = torch.device(device)
    B, S, M, C = value.shape
    Q = ref.shape[1]
    if shared:
        off = off.reshape(1, Q, M, -1).expand(B, -1, -1, -1)
        logits = logits.reshape(1, Q, M, -1).expand(B, -1, -1, -1)
    mk = mask.detach().to(dev, F64).reshape(B, Q, 1, 1)
    go = None
    if grad_slots is not None:
        go = mk * grad_slots.detach().to(dev, F64).reshape(1, Q, M, C)
    per = msda_f64(value, shapes, ref, off, logits, go, device=device)
    o = per["out"]
    slots = lambda t: t.sum(0).reshape(Q, M * C)  # noqa: E731
    e32 = (8 + o["n"]) * 2.0**-24 * o["mag"] + 2.0**-24 * o["pmag"]
    res = {"out": _entry(slots(mk * o["r"]), slots(mk.abs() * o["mag"]), o["n"].amax(0).reshape(Q, M * C) + B + 1,
                         slots(mk.abs() * o["pmag"]), slots(mk.abs() * (o["r"].abs() + e32)),
                         slots(mk.abs().expand_as(o["r"])))}  # fmt: skip
    if go is not None:
        ones = msda_f64(value, shapes, ref, off, logits, (go != 0).to(F64), index=None, device=device)
        for name in ("grad_value", "grad_ref", "grad_off", "grad_logits"):
            e, e1 = per[name], ones[name]
            e = _entry(e["r"], e["mag"], e["n"], e["pmag"], e["mag"], e1["mag"])
            if shared and name in ("grad_off", "grad_logits"):
                sm = lambda t: t.sum(0, keepdim=True)  # noqa: E731
                e = _entry(sm(e["r"]), sm(e["mag"]), e["n"].amax(0, keepdim=True) + B, sm(e["pmag"]),
                           (2 + 2.0**-6) * sm(e["mag"]), sm(e1["mag"]) + B)  # fmt: skip
            res[name] = e
    return res


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def dcn_f64(x, offset, mask, weight, bias, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, grad_out=None,
            device="cpu"):
    """Modulated deformable convolution (mmcv's DCNv2): x [N,C,H,W], offset [N, dg*2*kh*kw, Ho, Wo] ((dh, dw) pairs per
    tap), mask [N, dg*kh*kw, Ho, Wo], weight [Co, C/groups, kh, kw], bias [Co] or None, grad_out [N,Co,Ho,Wo] or None.
    Returns {"out": entry} and, with grad_out, "grad_input", "grad_offset", "grad_mask", "grad_weight" and (with a bias)
    "grad_bias" entries in the inputs' shapes (float64 on ``device``)."""
    dev = torch.device(device)
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    N, C, H, W = x.shape
    Co, cg, kh, kw = weight.shape
    g, dg, kk = groups, deform_groups, kh * kw
    Ho, Wo = offset.shape[2:]
    P, cpd, Mg = Ho * Wo, C // dg, Co // groups
    ti = torch.arange(kh, device=dev).repeat_interleave(kw)
    tj = torch.arange(kw, device=dev).repeat(kh)
    base_h = (torch.arange(Ho, device=dev) * sh - ph)[None, :, None] + (ti * dh)[:, None, None]  # [kk, Ho, 1]
    base_w = (torch.arange(Wo, device=dev) * sw - pw)[None, None, :] + (tj * dw)[:, None, None]  # [kk, 1, Wo]
    o32 = offset.detach().to(dev, torch.float32).reshape(N, dg, kk, 2, Ho, Wo)
    pos_h = (o32[:, :, :, 0] + base_h.float()).double().reshape(N, dg, kk, P)  # the fp32 sums the kernels form
    pos_w = (o32[:, :, :, 1] + base_w.float()).double().reshape(N, dg, kk, P)
    ok = (pos_h > -1) & (pos_w > -1) & (pos_h < H) & (pos_w < W)
    hl, wl = pos_h.floor(), pos_w.floor()
    lh, lw = pos_h - hl, pos_w - wl
    hh, hw_ = 1 - lh, 1 - lw
    hl, wl = hl.long(), wl.long()
    valid = torch.stack([ok & (hl + dy >= 0) & (hl + dy <= H - 1) & (wl + dx >= 0) & (wl + dx <= W - 1) for dy, dx in _TAPS])
    wts = torch.stack([hh * hw_, hh * lw, lh * hw_, lh * lw]) * valid  # [4, N, dg, kk, P]
    pix = torch.stack([(hl + dy).clamp(0, H - 1) * W + (wl + dx).clamp(0, W - 1) for dy, dx in _TAPS])
    x64 = x.detach().to(dev, F64).reshape(N, dg, cpd, H * W)
    idx = pix.reshape(4, N, dg, 1, kk * P).expand(4, N, dg, cpd, kk * P)
    xt = torch.stack([x64.gather(3, idx[t]) for t in range(4)]).reshape(4, N, dg, cpd, kk, P) * valid.unsqueeze(3)
    xa = xt.abs()
    w4 = wts.unsqueeze(3)  # [4, N, dg, 1, kk, P]
    m64 = mask.detach().to(dev, F64).reshape(N, dg, 1, kk, P)
    bil, bila = (w4 * xt).sum(0), (w4 * xa).sum(0)  # [N, dg, cpd, kk, P]
    col, cola = (m64 * bil).reshape(N, g, cg, kk, P), (m64.abs() * bila).reshape(N, g, cg, kk, P)
    w64 = weight.detach().to(dev, F64).reshape(g, Mg, cg, kk)
    out = torch.einsum("gmct,ngctp->ngmp", w64, col).reshape(N, Co, P)
    mag = torch.einsum("gmct,ngctp->ngmp", w64.abs(), cola).reshape(N, Co, P)
    if bias is not None:
        b64 = bias.detach().to(dev, F64).view(1, Co, 1)
        out, mag = out + b64, mag + b64.abs()
    # the fused FP16 kernel (csrc/dcn_fused.cu:337-354) blends each column in FP16: the four weights mask x bilinear are
    # rounded to FP16, then one __hmul2 and three __hfma2, five roundings of values at most |mask| sum_t w_t |x_t|
    # (counted as 6 to cover their second-order terms); subnormal weights or partial sums err by half the smallest
    # subnormal each: once per corner value read (times |x_t|) and once per operation
    vcnt = (xa.sum(0) + 4).reshape(N, g, cg, kk, P)
    lmag = 6 * torch.einsum("gmct,ngctp->ngmp", w64.abs(), cola).reshape(N, Co, Ho, Wo)
    lcnt = torch.einsum("gmct,ngctp->ngmp", w64.abs(), vcnt).reshape(N, Co, Ho, Wo)
    res = {"out": _entry(out.reshape(N, Co, Ho, Wo), mag.reshape(N, Co, Ho, Wo), cg * kk + 9, lmag=lmag, lcnt=lcnt)}
    if grad_out is None:
        return res
    go = grad_out.detach().to(dev, F64).reshape(N, g, Mg, P)
    ga = go.abs()
    gc = torch.einsum("gmct,ngmp->ngctp", w64, go).reshape(N, dg, cpd, kk, P)  # W^T grad_out per (channel, tap, pixel)
    gca = torch.einsum("gmct,ngmp->ngctp", w64.abs(), ga).reshape(N, dg, cpd, kk, P)
    if bias is not None:
        res["grad_bias"] = _entry(go.sum((0, 3)).reshape(Co), ga.sum((0, 3)).reshape(Co), N * P)
    res["grad_weight"] = _entry(torch.einsum("ngmp,ngctp->gmct", go, col).reshape(Co, cg, kh, kw),
                                torch.einsum("ngmp,ngctp->gmct", ga, cola).reshape(Co, cg, kh, kw), N * P + 9)
    ms = (N, dg * kk, Ho, Wo)
    res["grad_mask"] = _entry((gc * bil).sum(2).reshape(ms), (gca * bila).sum(2).reshape(ms), cpd + Mg + 9)
    m = m64  # [N, dg, 1, kk, P]
    dh_r = hw_.unsqueeze(2) * (xt[2] - xt[0]) + lw.unsqueeze(2) * (xt[3] - xt[1])
    dw_r = hh.unsqueeze(2) * (xt[1] - xt[0]) + lh.unsqueeze(2) * (xt[3] - xt[2])
    dh_m = hw_.unsqueeze(2) * (xa[2] + xa[0]) + lw.unsqueeze(2) * (xa[3] + xa[1])
    dw_m = hh.unsqueeze(2) * (xa[1] + xa[0]) + lh.unsqueeze(2) * (xa[3] + xa[2])
    okc = ok.unsqueeze(2)
    goff_r = torch.stack([((gc * m * dh_r) * okc).sum(2), ((gc * m * dw_r) * okc).sum(2)], 3)  # [N, dg, kk, 2, P]
    goff_m = torch.stack([((gca * m.abs() * dh_m) * okc).sum(2), ((gca * m.abs() * dw_m) * okc).sum(2)], 3)
    os_ = (N, dg * 2 * kk, Ho, Wo)
    res["grad_offset"] = _entry(goff_r.reshape(os_), goff_m.reshape(os_), cpd + Mg + 9)
    gi = torch.zeros(N, dg, cpd, H * W, dtype=F64, device=dev)
    gia = torch.zeros_like(gi)
    cnt = torch.zeros(N, dg, 1, H * W, dtype=F64, device=dev)
    for t in range(4):
        contrib = (gc * m * wts[t].unsqueeze(2)).reshape(N, dg, cpd, kk * P)
        gi.scatter_add_(3, idx[t], contrib)
        gia.scatter_add_(3, idx[t], (gca * m.abs() * wts[t].unsqueeze(2)).reshape(N, dg, cpd, kk * P))
        cnt.scatter_add_(3, idx[t][:, :, :1], valid[t].reshape(N, dg, 1, kk * P).to(F64))
    res["grad_input"] = _entry(gi.reshape(N, C, H, W), gia.reshape(N, C, H, W),
                               (cnt + Mg + 9).expand(N, dg, cpd, H * W).reshape(N, C, H, W))
    return res


def rotate_f64(img, ix, iy, interp):
    """RotateTRT's sampling step: img [C, H, W] (the values the kernel reads: FP16 values widened, or the fp32 products
    q * scale_i for INT8), ix / iy [H, W] the source index of every output pixel (float32, as the kernel forms them).
    Bilinear (interp 0): the four taps around (ix, iy) weighted (x1 - ix)(y1 - iy), (ix - x0)(y1 - iy),
    (x1 - ix)(iy - y0), (ix - x0)(iy - y0) in float64, a tap outside the image contributing 0; n = 4. Nearest
    (interp 1): the pixel at round-half-away-from-zero (ix, iy) (roundf), 0 outside; n = 1. Same entry as above, on the
    device of ``img``; mag = sum |w_i v_i|."""
    v = img.detach().to(F64)
    C, H, W = v.shape
    flat = v.reshape(C, H * W)
    x, y = ix.detach().to(v.device, F64), iy.detach().to(v.device, F64)

    def tap(xi, yi):
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        pix = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long().reshape(-1)
        return flat[:, pix].reshape(C, H, W) * ok

    if interp == 1:
        rnd = lambda t: torch.sign(t) * torch.floor(t.abs() + 0.5)  # noqa: E731
        r = tap(rnd(x), rnd(y))
        return _entry(r, r.abs(), 1)
    x0, y0 = x.floor(), y.floor()
    x1, y1 = x0 + 1, y0 + 1
    r = torch.zeros(C, H, W, dtype=F64, device=v.device)
    mag = torch.zeros_like(r)
    for xi, yi, w in ((x0, y0, (x1 - x) * (y1 - y)), (x1, y0, (x - x0) * (y1 - y)), (x0, y1, (x1 - x) * (y - y0)),
                      (x1, y1, (x - x0) * (y - y0))):  # fmt: skip
        t = tap(xi, yi) * w
        r += t
        mag += t.abs()
    return _entry(r, mag, 4)
