"""TEST INFRASTRUCTURE ONLY for the fp16 inference mode (precision="fp16"): torch-CPU emulations of what the single-pass
kernels compute, extending tests/emu_ops.py, so an fp16 engine can run without a GPU and a GPU run can be compared with the
same engine emulated.  Nothing under aot_benchmark_b200/ imports this module.

- conv2d / linear with a registered tensor-core weight, in an fp16 call: fp16(x) times the weight the kernel streams,
  fp16(w 2^e) 2^-e, summed in float32 (the kernel sums in fp32 too, in its own order).
- lt_attention_tc / gp_attention_tc with the exact bit clear: hi-only Q and K; P rounded to fp16 relative to the final row
  max of its split (the kernel rounds relative to the running max, so this is close, not bitwise); the row sum l and V
  (hi + lo) are unrounded."""
import torch

import emu_ops


def _ops():
    from aot_benchmark_b200 import ops
    return ops


def rounded_weight(w):
    """The fp32 [K, Cout] weight the single-pass kernel multiplies by for registered weight w, or None."""
    ops = _ops()
    t = ops._TC_WEIGHTS.get(w.data_ptr())
    if t is None or ops.CONV_IMPL != "tc":
        return None
    wh, _, ws = t[:3]
    r = wh[:, :w.shape[0]].float().t()
    if ws is not None:
        r = r * ws.float()                     # exact: powers of two
    return r.contiguous().to(w.device)


def _fp16_call(w):
    return _ops()._PRECISION == "fp16" and rounded_weight(w) is not None


def conv2d(x, w, bias, out, res=None, KH=1, KW=1, stride=1, pad=0, dil=1, act=0, stream=None):
    if dil == 1 and _fp16_call(w):
        return emu_ops.conv2d(x.half().float(), rounded_weight(w), bias, out, res, KH, KW, stride, pad, dil, act)
    return emu_ops.conv2d(x, w, bias, out, res, KH, KW, stride, pad, dil, act)


def linear(x, wt, bias, out, res=None, act=0, stream=None):
    if _fp16_call(wt):
        return emu_ops.linear(x.half().float(), rounded_weight(wt), bias, out, res, act)
    return emu_ops.linear(x, wt, bias, out, res, act)


def _split_parts(q, k, v, tk, splits, tile, exact):
    """Per split: (P V, m, l) over keys [z per tile, (z + 1) per tile) with q [.., N, d], k / v [.., tk, d]."""
    tiles = (tk + tile - 1) // tile
    per = (tiles + splits - 1) // splits
    parts = []
    for z in range(splits):
        k0, k1 = min(z * per * tile, tk), min((z + 1) * per * tile, tk)
        if k1 <= k0:
            parts.append(None)
            continue
        s = q @ k[..., k0:k1, :].transpose(-1, -2)
        m = s.max(-1).values
        p = torch.exp(s - m.unsqueeze(-1))
        pv = p if exact else p.half().float()
        parts.append((pv @ v[..., k0:k1, :], m, p.sum(-1)))
    return parts


def lt_attention_tc(Qp, Kp, Vp, N, Tk, O=None, Tk_dev=None, splits=1, exact=True, part=None, dbg=None, stream=None,
                    merge=True, variant=None):
    if exact:
        return emu_ops.lt_attention_tc(Qp, Kp, Vp, N, Tk, O, Tk_dev, splits, exact, part, dbg, stream, merge, variant)
    tk = int(Tk_dev.item()) if Tk_dev is not None else int(Tk)
    Hh = Qp.shape[0]
    q, k = Qp[:, :N, :32].float(), Kp[:, :tk, :32].float()
    v = Vp[:, :tk, :32].float() + Vp[:, :tk, 32:].float()
    parts = _split_parts(q, k, v, tk, splits, 128, exact)
    empty = (torch.zeros(Hh, N, 32), torch.full((Hh, N), float("-inf")), torch.zeros(Hh, N))
    parts = [p if p is not None else empty for p in parts]
    if splits == 1:
        o, m, l = parts[0]
        O.copy_((o / l.unsqueeze(-1)).permute(1, 0, 2).reshape(N, Hh * 32))
        return O
    Op, Mp, Lp = part
    for z, (o, m, l) in enumerate(parts):
        Op[z].copy_(o.permute(1, 0, 2).reshape(N, Hh * 32))
        Mp[z].copy_(m)
        Lp[z].copy_(l)
    if merge:
        emu_ops.attn_merge(Op, Mp, Lp, O, Hh, 32)
    return O


def gp_attention_tc(Qp, Kp, Vp, N, Tk, O=None, Tk_dev=None, splits=1, exact=True, part=None, stream=None, merge=True):
    if exact:
        return emu_ops.gp_attention_tc(Qp, Kp, Vp, N, Tk, O, Tk_dev, splits, exact, part, stream, merge)
    tk = int(Tk_dev.item()) if Tk_dev is not None else int(Tk)
    unpack = lambda P, rows, lo: (P[:, :rows, :32].float() + (P[:, :rows, 32:].float() if lo else 0)) \
        .permute(1, 0, 2).reshape(rows, -1)
    q, k, v = unpack(Qp, N, False), unpack(Kp, tk, False), unpack(Vp, tk, True)
    dv = v.shape[1]
    parts = _split_parts(q, k, v, tk, splits, 64, exact)
    empty = (torch.zeros(N, dv), torch.full((N,), float("-inf")), torch.zeros(N))
    parts = [p if p is not None else empty for p in parts]
    if splits == 1:
        o, m, l = parts[0]
        O.copy_(o / l.unsqueeze(-1))
        return O
    Op, Mp, Lp = part
    for z, (o, m, l) in enumerate(parts):
        Op[z].copy_(o)
        Mp[z, 0].copy_(m)
        Lp[z, 0].copy_(l)
    if merge:
        emu_ops.attn_merge(Op, Mp, Lp, O, 1, dv)
    return O


EMULATED = ("conv2d", "linear", "lt_attention_tc", "gp_attention_tc")


def install_engine(monkeypatch, bounded=False):
    """emu_ops.install_engine (plus the bounded bank's entry points if `bounded`) with the fp16-aware emulations."""
    from aot_benchmark_b200 import ops
    if bounded:
        import bounded_bank_support
        bounded_bank_support.install_engine(monkeypatch)
    else:
        emu_ops.install_engine(monkeypatch)
    for name in EMULATED:
        monkeypatch.setattr(ops, name, globals()[name])


def build_engine(model_name, sd, gap, precision, device="cpu", **kw):
    """The product engine of `model_name` (eval phase) on a model with state dict `sd`."""
    from aot_benchmark_b200 import EngineConfig, build_engine as _build, build_vos_model
    cfg = EngineConfig("t", model_name)
    model = build_vos_model(cfg.MODEL_VOS, cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(device).eval()
    eng = _build(cfg.MODEL_ENGINE, phase="eval", aot_model=model, gpu_id=0, long_term_mem_gap=gap,
                 short_term_mem_skip=cfg.TEST_SHORT_TERM_MEM_SKIP, precision=precision, **kw)
    eng.eval()
    return eng
