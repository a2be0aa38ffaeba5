"""Tensor-level wrappers over the C ABI (torch is used for device memory and streams only).

Every function enqueues on torch's current CUDA stream and returns its outputs; there is
no eager/CPU implementation behind these calls.
"""
import ctypes
import math

import torch

from big_vision_b200 import lib as L

_DT = {torch.float32: L.F32, torch.bfloat16: L.BF16}


def _dt(t):
  try:
    return _DT[t.dtype]
  except KeyError:
    raise L.BvError(f"unsupported dtype {t.dtype}") from None


def _p(t):
  if t is None:
    return None
  if not t.is_cuda:
    raise L.BvError("bv_b200 kernels need CUDA tensors (no CPU fallback)")
  return ctypes.c_void_p(t.data_ptr())


def _stream():
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rowmajor(t):
  """Returns (tensor, ld) for a 2-D tensor whose last dim is contiguous."""
  assert t.dim() == 2 and t.stride(1) == 1, (t.shape, t.stride())
  return t, t.stride(0)


def gemm(a, b, *, a_mn=False, b_mn=False, out=None, out_dtype=torch.bfloat16, bias=None,
         aux=None, aux_row_mod=0, epilogue=None, out2=None, reduce_out=False, splits=0,
         block_n=0, alpha=1.0, M=None, N=None, K=None, colsum=None):
  """D[M,N] = epi(alpha * A.B^T) with A,B given as STORED 2-D tensors.

  a_mn=False: a is [M,K]; a_mn=True: a is [K,M].  Same for b with N.
  """
  a, lda = _rowmajor(a)
  b, ldb = _rowmajor(b)
  if M is None:
    M = a.shape[1] if a_mn else a.shape[0]
  if K is None:
    K = a.shape[0] if a_mn else a.shape[1]
  if N is None:
    N = b.shape[1] if b_mn else b.shape[0]
  kb = b.shape[0] if b_mn else b.shape[1]
  assert kb >= K or kb == K, (a.shape, b.shape, a_mn, b_mn)
  if out is None:
    out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    if reduce_out:
      out.zero_()
  out, ldd = _rowmajor(out)
  if epilogue is None:
    epilogue = L.EPI_BIAS if bias is not None else L.EPI_NONE
  ldd2 = 0
  if epilogue == L.EPI_BIAS_GELU:
    if out2 is None:
      out2 = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
    out2, ldd2 = _rowmajor(out2)
  ldaux = 0
  if aux is not None:
    aux, ldaux = _rowmajor(aux)
  args = L.GemmArgs(
      A=a.data_ptr(), B=b.data_ptr(), D=out.data_ptr(),
      D2=out2.data_ptr() if out2 is not None else None,
      bias=bias.data_ptr() if bias is not None else None,
      aux=aux.data_ptr() if aux is not None else None,
      colsum=colsum.data_ptr() if colsum is not None else None,
      M=M, N=N, K=K, lda=lda, ldb=ldb, ldd=ldd, ldd2=ldd2, ldaux=ldaux,
      a_mn=int(a_mn), b_mn=int(b_mn), epilogue=epilogue, out_dtype=_dt(out),
      reduce_out=int(reduce_out), splits=splits, block_n=block_n, aux_row_mod=aux_row_mod,
      alpha=alpha)
  for t in (a, b, out):
    if not t.is_cuda:
      raise L.BvError("bv_gemm needs CUDA tensors")
  tag = None
  if L.PROFILE is not None:       # bench.py --profile-calls: one line per GEMM shape
    tag = (f"bv_gemm {M}x{N}x{K} {'T' if a_mn else 'N'}{'T' if b_mn else 'N'} epi{epilogue}"
           f"{' f32' if out.dtype == torch.float32 else ''}{' red' if reduce_out else ''}", 2.0 * M * N * K)
  L.call("bv_gemm", ctypes.byref(args), _stream(), tag=tag)
  if epilogue == L.EPI_BIAS_GELU:
    return out, out2
  return out


def layernorm_fwd(x, scale, bias, *, out_dtype=torch.bfloat16, eps=1e-6):
  rows, d = x.shape
  y = torch.empty((rows, d), dtype=out_dtype, device=x.device)
  mean = torch.empty((rows,), dtype=torch.float32, device=x.device)
  rstd = torch.empty((rows,), dtype=torch.float32, device=x.device)
  L.call("bv_layernorm_fwd", _p(x), _dt(x), _p(scale), _p(bias), _p(y), _dt(y), _p(mean), _p(rstd),
         rows, d, eps, _stream())
  return y, mean, rstd


def layernorm_bwd(dy, x, scale, mean, rstd, *, dres=None, dx_dtype=torch.bfloat16, dscale=None,
                  dbias=None, dx_colsum=None):
  rows, d = x.shape
  dx = torch.empty((rows, d), dtype=dx_dtype, device=x.device)
  if dres is not None:
    assert dres.dtype == dx_dtype and dres.is_contiguous()
  L.call("bv_layernorm_bwd", _p(dy), _dt(dy), _p(x), _dt(x), _p(scale), _p(mean), _p(rstd),
         _p(dres), _p(dx), _dt(dx), _p(dscale), _p(dbias), _p(dx_colsum), rows, d, _stream())
  return dx


def _attn_view(t):
  """t: [B, N, cols] view with unit stride on the last dim -> (ptr, ld, bs)."""
  assert t.dim() == 3 and t.stride(2) == 1, (t.shape, t.stride())
  return t.data_ptr(), t.stride(1), t.stride(0)


def _attn_args(q, k, v, o, lse, heads, scale):
  B, Nq, _ = q.shape
  Nk = k.shape[1]
  qp, ldq, bsq = _attn_view(q)
  kp, ldk, bsk = _attn_view(k)
  vp, ldv, bsv = _attn_view(v)
  op, ldo, bso = _attn_view(o)
  return L.AttnArgs(q=qp, k=kp, v=vp, o=op, lse=lse.data_ptr(), B=B, H=heads, Nq=Nq, Nk=Nk,
                    ldq=ldq, ldk=ldk, ldv=ldv, ldo=ldo, bsq=bsq, bsk=bsk, bsv=bsv, bso=bso,
                    scale=scale)


def _attn_call(name, args, masked_type, key_mask, B, Nk, dh, dropout=None, dropout_type=None):
  """Calls `name` on `args`; with a key mask, on a `masked_type` that appends it, and head_dim | ATTN_KEY_MASK
  (the arguments are its first member, so the pointer is the same); with a dropout key too, on a
  `dropout_type` that appends the key to that, and head_dim | ATTN_KEY_MASK | ATTN_DROPOUT."""
  if key_mask is None:
    if dropout is not None:
      raise L.BvError("attention: dropout is built for key-masked attention only; pass a key_mask")
    L.call(name, ctypes.byref(args), dh, _stream())
    return
  if key_mask.dtype not in (torch.uint8, torch.bool) or tuple(key_mask.shape) != (B, Nk) or key_mask.stride(1) != 1:
    raise L.BvError(f"attention: key_mask must be uint8 or bool [B, Nk] = [{B}, {Nk}] with unit key stride, got "
                    f"{key_mask.dtype} {tuple(key_mask.shape)}")
  m = masked_type(attn=args, key_mask=_p(key_mask), bsmask=key_mask.stride(0))
  if dropout is None:
    L.call(name, ctypes.byref(m.attn), dh | L.ATTN_KEY_MASK, _stream())
    return
  d = dropout_type(masked=m, drop=dropout)
  L.call(name, ctypes.byref(d.masked.attn), dh | L.ATTN_KEY_MASK | L.ATTN_DROPOUT, _stream())


# head dims the attention kernels are built for (bv_attention_fwd_hd / bv_attention_bwd_hd)
ATTN_HEAD_DIMS = (64, 72, 80, 96, 104)


def _head_dim(cols, heads):
  if cols % heads:
    raise ValueError(f"attention: {cols} columns do not split into {heads} heads")
  return cols // heads


def attention_fwd(q, k, v, heads, scale=None, key_mask=None, dropout=None):
  """q:[B,Nq,H*dh] k,v:[B,Nk,H*dh] bf16 (strided views allowed) -> o [B,Nq,H*dh], lse [B,H,Nq].

  dh is one of ATTN_HEAD_DIMS; the library refuses any other.  key_mask: None, or uint8 / bool [B, Nk],
  nonzero = attend (head dim 64 only); a query with every key masked gets o = 0 and lse = 0.  dropout: None, or
  the lib.DropoutKey of attention-probability dropout (with a key_mask only; row0 = the global index of sample 0
  times H * Nq, include/bv_dropout.h); lse stays that of the undropped softmax."""
  B, Nq, cols = q.shape
  dh = _head_dim(cols, heads)
  if scale is None:
    scale = 1.0 / math.sqrt(dh)
  o = torch.empty((B, Nq, cols), dtype=torch.bfloat16, device=q.device)
  lse = torch.empty((B, heads, Nq), dtype=torch.float32, device=q.device)
  args = _attn_args(q, k, v, o, lse, heads, scale)
  _attn_call("bv_attention_fwd_hd", args, L.AttnMaskedArgs, key_mask, B, k.shape[1], dh, dropout, L.AttnDropoutArgs)
  return o, lse


def attention_bwd(do, q, k, v, o, lse, heads, scale=None, dq=None, dk=None, dv=None,
                  dq_colsum=None, dk_colsum=None, dv_colsum=None, key_mask=None, dropout=None):
  """Gradients of attention_fwd (the same key_mask and dropout key): -> dq, dk, dv; masked keys get dk = dv = 0."""
  dh = _head_dim(q.shape[2], heads)
  if scale is None:
    scale = 1.0 / math.sqrt(dh)
  if dq is None:
    dq = torch.empty(q.shape, dtype=torch.bfloat16, device=q.device)
  if dk is None:
    dk = torch.empty(k.shape, dtype=torch.bfloat16, device=q.device)
  if dv is None:
    dv = torch.empty(v.shape, dtype=torch.bfloat16, device=q.device)
  f = _attn_args(q, k, v, o, lse, heads, scale)
  B, Nq, _ = q.shape
  delta = torch.empty((B, heads, Nq), dtype=torch.float32, device=q.device)
  dop, lddo, bsdo = _attn_view(do)
  dqp, lddq, bsdq = _attn_view(dq)
  dkp, lddk, bsdk = _attn_view(dk)
  dvp, lddv, bsdv = _attn_view(dv)
  args = L.AttnBwdArgs(fwd=f, d_o=dop, lddo=lddo, bsdo=bsdo, dq=dqp, dk=dkp, dv=dvp,
                       lddq=lddq, lddk=lddk, lddv=lddv, bsdq=bsdq, bsdk=bsdk, bsdv=bsdv,
                       dq_colsum=dq_colsum.data_ptr() if dq_colsum is not None else None,
                       dk_colsum=dk_colsum.data_ptr() if dk_colsum is not None else None,
                       dv_colsum=dv_colsum.data_ptr() if dv_colsum is not None else None,
                       delta=delta.data_ptr())
  _attn_call("bv_attention_bwd_hd", args, L.AttnMaskedBwdArgs, key_mask, B, k.shape[1], dh, dropout,
             L.AttnDropoutBwdArgs)
  return dq, dk, dv


def patchify(image, patch, value_range=(-1.0, 1.0), in_range=(0.0, 255.0), clip_values=False):
  """image [n,H,W,C]: fp32 (already in its value range) or uint8 (decoded pixels; `value_range(...)`
  of the input pipeline, pp/ops_general.py:32-64, is applied on the fly)."""
  n, H, W, C = image.shape
  assert image.is_contiguous()
  if image.dtype == torch.uint8:
    kp = (patch * patch * C + 7) // 8 * 8
    out = torch.empty((n * (H // patch) * (W // patch), kp), dtype=torch.bfloat16, device=image.device)
    L.call("bv_patchify_u8", _p(image), _p(out), n, H, W, C, patch, float(value_range[0]),
           float(value_range[1]), float(in_range[0]), float(in_range[1]), int(clip_values), _stream())
    return out
  assert image.dtype == torch.float32
  kp = (patch * patch * C + 7) // 8 * 8
  out = torch.empty((n * (H // patch) * (W // patch), kp), dtype=torch.bfloat16, device=image.device)
  L.call("bv_patchify", _p(image), _p(out), n, H, W, C, patch, _stream())
  return out


def embed_fwd(ids, table, pos, out_dtype=torch.bfloat16):
  n, Ln = ids.shape
  vocab, d = table.shape
  assert ids.dtype == torch.int32 and ids.is_contiguous()
  out = torch.empty((n * Ln, d), dtype=out_dtype, device=table.device)
  L.call("bv_embed_fwd", _p(ids), _p(table), _p(pos), _p(out), _dt(out), n, Ln, d, vocab, _stream())
  return out


def embed_bwd(ids, dy, dtable, dpos):
  n, Ln = ids.shape
  vocab, d = dtable.shape
  L.call("bv_embed_bwd", _p(ids), _p(dy), _dt(dy), _p(dtable), _p(dpos), n, Ln, d, vocab, _stream())


def colsum(x, out):
  x, ld = _rowmajor(x)
  L.call("bv_colsum", _p(x), _dt(x), _p(out), x.shape[0], x.shape[1], ld, _stream())
  return out


def cast(src, dst):
  assert src.is_contiguous() and dst.is_contiguous() and src.numel() == dst.numel()
  L.call("bv_cast", _p(src), _dt(src), _p(dst), _dt(dst), src.numel(), _stream())
  return dst


def l2norm_fwd(x, eps=1e-8):
  n, d = x.shape
  z = torch.empty((n, d), dtype=torch.float32, device=x.device)
  norm = torch.empty((n,), dtype=torch.float32, device=x.device)
  L.call("bv_l2norm_fwd", _p(x), _dt(x), _p(z), _p(norm), n, d, eps, _stream())
  return z, norm


def l2norm_bwd(dz, z, norm, dx_dtype=torch.float32, eps=1e-8):
  n, d = z.shape
  dx = torch.empty((n, d), dtype=dx_dtype, device=z.device)
  L.call("bv_l2norm_bwd", _p(dz), _p(z), _p(norm), _p(dx), _dt(dx), n, d, eps, _stream())
  return dx


def pool_fwd(x, n, N, mode, tok=0, out_dtype=None):
  d = x.shape[-1]
  y = torch.empty((n, d), dtype=out_dtype or x.dtype, device=x.device)
  L.call("bv_pool_fwd", _p(x), _dt(x), _p(y), _dt(y), n, N, d, mode, tok, _stream())
  return y


def pool_bwd(dy, n, N, mode, tok=0, dx_dtype=torch.bfloat16):
  d = dy.shape[-1]
  dx = torch.empty((n * N, d), dtype=dx_dtype, device=dy.device)
  L.call("bv_pool_bwd", _p(dy), _dt(dy), _p(dx), _dt(dx), n, N, d, mode, tok, _stream())
  return dx


def pool_max_bwd(dy, x, n, N, dx_dtype=torch.bfloat16):
  d = dy.shape[-1]
  dx = torch.empty((n * N, d), dtype=dx_dtype, device=dy.device)
  L.call("bv_pool_max_bwd", _p(dy), _dt(dy), _p(x), _dt(x), _p(dx), _dt(dx), n, N, d, _stream())
  return dx


def broadcast_row(x, rows, row=None, out_dtype=None):
  d = x.shape[-1]
  y = torch.empty((rows, d), dtype=out_dtype or x.dtype, device=x.device)
  L.call("bv_broadcast_row", _p(x), _dt(x), _p(row), _p(y), _dt(y), rows, d, _stream())
  return y


def tanh_fwd(x):
  y = torch.empty_like(x)
  L.call("bv_tanh_fwd", _p(x), _p(y), _dt(x), x.numel(), _stream())
  return y


def tanh_bwd(dy, y):
  dx = torch.empty_like(y)
  L.call("bv_tanh_bwd", _p(dy), _p(y), _p(dx), _dt(y), y.numel(), _stream())
  return dx


def gelu_fwd(x):
  y = torch.empty_like(x)
  L.call("bv_gelu_fwd", _p(x), _p(y), _dt(x), x.numel(), _stream())
  return y


def mixup(x, a):
  """a * x + (1 - a) * roll(x, 1, axis 0) for an fp32 tensor (rows of any length)."""
  x = x.contiguous()
  assert x.dtype == torch.float32, x.dtype
  out = torch.empty_like(x)
  n = x.shape[0]
  L.call("bv_mixup", _p(x), _p(out), n, x.numel() // n, float(a), _stream())
  return out


def axpby(x, y, a=1.0, b=1.0, out=None):
  if out is None:
    out = torch.empty_like(x)
  L.call("bv_axpby", _p(x), _p(y), _p(out), _dt(x), a, b, x.numel(), _stream())
  return out


def transpose_tokens(x, n, N, d):
  npad = (N + 7) // 8 * 8
  y = torch.empty((n * d, npad), dtype=torch.bfloat16, device=x.device)
  L.call("bv_transpose_tokens", _p(x), _p(y), n, N, d, _stream())
  return y


def untranspose_add(y, res, n, N, d):
  out = torch.empty((n * N, d), dtype=torch.bfloat16, device=y.device)
  L.call("bv_untranspose_add", _p(y), _p(res), _p(out), n, N, d, _stream())
  return out


def row_select(a, b, mask, n, N):
  """out[b,t,:] = mask[b] != 0 ? a[b,t,:] : (b[b,t,:] or 0): the stochastic-depth residual gate."""
  d = a.shape[-1]
  assert a.dtype == torch.bfloat16 and a.is_contiguous() and mask.dtype == torch.float32
  out = torch.empty_like(a)
  L.call("bv_row_select", _p(a), _p(b), _p(mask), _p(out), n, N, d, _stream())
  return out


def concat_cls(x, cls, n, N0):
  d = x.shape[-1]
  out = torch.empty((n * (N0 + 1), d), dtype=torch.bfloat16, device=x.device)
  L.call("bv_concat_cls", _p(x), _p(cls), _p(out), n, N0, d, _stream())
  return out


def drop_cls(x, n, N0):
  d = x.shape[-1]
  out = torch.empty((n * N0, d), dtype=torch.bfloat16, device=x.device)
  L.call("bv_drop_cls", _p(x), _p(out), n, N0, d, _stream())
  return out


def _bf16_2d(*ts):
  for t in ts:
    if t.dtype != torch.bfloat16 or t.dim() != 2 or t.stride(1) != 1:
      raise L.BvError(f"dropout takes bf16 [rows, cols] matrices with a contiguous last axis, got "
                      f"{t.dtype} {tuple(t.shape)} {t.stride()}")


def dropout(x, key, out=None, colsum_into=None):
  """out = dropout(x) under `key` (lib.DropoutKey) for bf16 [rows, cols] (row-strided views allowed; `out`
  may be x).  colsum_into: None, or fp32 [cols] += the column sums of out (a bias gradient).  Returns out."""
  out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if out is None else out
  _bf16_2d(x, out)
  assert out.shape == x.shape, (tuple(x.shape), tuple(out.shape))
  L.call("bv_dropout", _p(x), x.stride(0), _p(out), out.stride(0), x.shape[0], x.shape[1], ctypes.byref(key),
         _stream())
  if colsum_into is not None:
    colsum(out, colsum_into)
  return out


def dropout_add(resid, y, key, out=None):
  """out = resid + dropout(y) under `key` for bf16 [rows, cols] (row-strided views allowed; `out` may be
  resid or y).  Returns out."""
  out = torch.empty(y.shape, dtype=torch.bfloat16, device=y.device) if out is None else out
  _bf16_2d(resid, y, out)
  assert resid.shape == y.shape == out.shape, (tuple(resid.shape), tuple(y.shape), tuple(out.shape))
  L.call("bv_dropout_add", _p(resid), resid.stride(0), _p(y), y.stride(0), _p(out), out.stride(0), y.shape[0],
         y.shape[1], ctypes.byref(key), _stream())
  return out


def siglip_loss(dots, row_offset, t_param, b_param, global_b, loss, dt, db):
  n, B = dots.shape
  # G feeds two GEMMs through TMA: its row stride must be a multiple of 16 bytes (8 bf16) even when the
  # slab is narrow (the chunked loss on a tiny per-rank batch: [4, 4])
  G = torch.empty((n, (B + 7) // 8 * 8), dtype=torch.bfloat16, device=dots.device)[:, :B]
  # per-block partials + fixed-order finishing pass: the scalars are run-to-run deterministic
  ws = torch.empty(L.LOSS_WS_FLOATS, dtype=torch.float32, device=dots.device)
  L.call("bv_siglip_loss", _p(dots), n, B, dots.stride(0), row_offset, _p(t_param), _p(b_param),
         global_b, _p(G), G.stride(0), _p(loss), _p(dt), _p(db), _p(ws), _stream())
  return G


def softmax_contrastive_loss(dots, row_offset, t_param, global_b, weight, loss, dt, ncorrect):
  """One direction of the CLIP softmax loss on dots [n, B]; returns G (bf16) = d loss / d dots."""
  n, B = dots.shape
  G = torch.empty((n, (B + 7) // 8 * 8), dtype=torch.bfloat16, device=dots.device)[:, :B]
  ws = torch.empty(3 * n, dtype=torch.float32, device=dots.device)
  L.call("bv_softmax_contrastive_loss", _p(dots), n, B, dots.stride(0), row_offset, _p(t_param), global_b,
         float(weight), _p(G), G.stride(0), _p(loss), _p(dt), _p(ncorrect), _p(ws), _stream())
  return G


def _xent(name, logits, labels, loss, want_grad, dlogits_cols):
  logits, ldx = _rowmajor(logits)
  labels, ldy = _rowmajor(labels)
  n, C = logits.shape
  dl = torch.empty((n, dlogits_cols or C), dtype=torch.float32, device=logits.device) if want_grad else None
  ws = torch.empty(n, dtype=torch.float32, device=logits.device)
  L.call(name, _p(logits), ldx, _p(labels), ldy, _p(loss), _p(dl), dl.stride(0) if want_grad else C, _p(ws), n, C,
         _stream())
  return dl


def sigmoid_xent(logits, labels, loss, want_grad=True, dlogits_cols=None):
  """Mean sigmoid cross-entropy of logits / labels [n, C] (row-strided views allowed) accumulated into
  `loss`; returns d loss / d logits [n, dlogits_cols or C], zero in the columns past C."""
  return _xent("bv_sigmoid_xent_ld", logits, labels, loss, want_grad, dlogits_cols)


def softmax_xent(logits, labels, loss, want_grad=True, dlogits_cols=None):
  """softmax_xent counterpart of sigmoid_xent."""
  return _xent("bv_softmax_xent_ld", logits, labels, loss, want_grad, dlogits_cols)


def sumsq(x, out):
  L.call("bv_sumsq", _p(x), _p(out), x.numel(), _stream())
  return out


def adam_step(params, grads, mu, nu, params_bf16, *, lr_eff, b1, b2, eps, wd_eff, step,
              grad_mult=1.0, clip_norm=0.0, gnorm_sq=None, upd_sq=None, param_sq=None):
  args = L.AdamArgs(
      params=params.data_ptr(), grads=grads.data_ptr(), mu=mu.data_ptr(), nu=nu.data_ptr(),
      params_bf16=params_bf16.data_ptr() if params_bf16 is not None else None,
      n=params.numel(), mu_dtype=_dt(mu), lr_eff=lr_eff, b1=b1, b2=b2, eps=eps, wd_eff=wd_eff,
      grad_mult=grad_mult, clip_norm=clip_norm,
      gnorm_sq=gnorm_sq.data_ptr() if gnorm_sq is not None else None, step=step,
      upd_sq=upd_sq.data_ptr() if upd_sq is not None else None,
      param_sq=param_sq.data_ptr() if param_sq is not None else None)
  L.call("bv_adam_step", ctypes.byref(args), _stream())


def scale_step(params, grads, params_bf16, *, lr_eff, wd_eff, grad_mult=1.0, clip_norm=0.0, gnorm_sq=None,
               upd_sq=None, param_sq=None):
  L.call("bv_scale_step", _p(params), _p(grads), _p(params_bf16), params.numel(), lr_eff, wd_eff, grad_mult,
         clip_norm, _p(gnorm_sq), _p(upd_sq), _p(param_sq), _stream())


def adafactor_step(P, tens, st, *, decay, eps, beta, lr_eff, wd_eff, grad_mult, clip_norm, gnorm_sq, upd_sq, param_sq):
  """One BV-Adafactor update of the reference tensor `tens` (optax._AdafactorTensor) in place."""
  A, Ld, M, H = tens.dims
  sA, sL, sM = tens.strides
  ptr = lambda buf: buf.data_ptr() + tens.offset * buf.element_size()
  opt = lambda k: st[k].data_ptr() if k in st else None
  args = L.AdafactorArgs(
      params=ptr(P.flat), grads=ptr(P.grad), params_bf16=ptr(P.half), A=A, L=Ld, M=M, H=H, sA=sA, sL=sL, sM=sM,
      mode=tens.mode, vfull=opt("vfull"), red_h=opt("red_h"), red_l=opt("red_l"), nrm=opt("nrm"),
      momentum=opt("momentum"), decay=decay, eps=eps, beta=beta, lr_eff=lr_eff, wd_eff=wd_eff,
      grad_mult=grad_mult, clip_norm=clip_norm, gnorm_sq=gnorm_sq.data_ptr(), upd_sq=upd_sq.data_ptr(),
      param_sq=param_sq.data_ptr())
  if not P.flat.is_cuda:
    raise L.BvError("bv_adafactor_step needs CUDA tensors")
  L.call("bv_adafactor_step", ctypes.byref(args), _stream())


# ---- GSAM / SAM (include/bv_b200_sam.h) --------------------------------------------------------
def _flat32(*ts):
  for t in ts:
    if t.dtype != torch.float32 or not t.is_contiguous():
      raise L.BvError(f"GSAM kernels take contiguous fp32 buffers, got {t.dtype}")


def sam_perturb(w, g, g_sumsq, rho, eps=1e-12, adaptive=False, out=None, out_bf16=None):
  """out = w + rho * g / (sqrt(g_sumsq) + eps) (times |w| with `adaptive`) and its bf16 shadow, in one pass;
  g_sumsq is a device scalar [1].  Returns (out, out_bf16)."""
  _flat32(w, g)
  out = torch.empty_like(w) if out is None else out
  out_bf16 = torch.empty(w.shape, dtype=torch.bfloat16, device=w.device) if out_bf16 is None else out_bf16
  assert out.numel() == out_bf16.numel() == g.numel() == w.numel() and out_bf16.dtype == torch.bfloat16
  L.call("bv_sam_perturb", _p(w), _p(g), _p(g_sumsq), float(rho), float(eps), int(bool(adaptive)), _p(out),
         _p(out_bf16), w.numel(), _stream())
  return out, out_bf16


def sam_dots(a, b, out=None, ws=None):
  """out [2] fp32 on the device = (a . b, b . b), summed in a fixed order (run-to-run identical)."""
  _flat32(a, b)
  assert a.numel() == b.numel()
  out = torch.empty(2, dtype=torch.float32, device=b.device) if out is None else out
  ws = torch.empty(L.SAM_WS_FLOATS, dtype=torch.float32, device=b.device) if ws is None else ws
  L.call("bv_sam_dots", _p(a), _p(b), _p(out), _p(ws), b.numel(), _stream())
  return out


def gsam_combine(g_clean, g_robust, dot, norm_sq, alpha, minimize_fp=True):
  """The GSAM gradient, in place over g_clean; dot = g_c . g_r and norm_sq (||g_r||^2 with minimize_fp,
  else ||g_c||^2) are device scalars [1]."""
  _flat32(g_clean, g_robust)
  assert g_clean.numel() == g_robust.numel()
  L.call("bv_gsam_combine", _p(g_clean), _p(g_robust), _p(dot), _p(norm_sq), float(alpha), int(bool(minimize_fp)),
         g_clean.numel(), _stream())
  return g_clean


# ---- distillation (include/bv_b200_distill.h) ------------------------------------------------------
def _logits2d(*ts):
  for t in ts:
    if t is not None and (t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1):
      raise L.BvError(f"distillation kernels take fp32 [n, C] matrices with a contiguous last axis, got "
                      f"{t.dtype} {tuple(t.shape)} {t.stride()}")


def distill_loss(student, teacher, labels=None, kind="kl", t=1.0, ls=0.0, dlogits=None, dlogits_cols=None,
                 want_grad=True):
  """One teacher's term of the distillation loss on logits [n, C] (row-strided views allowed).

  Returns (out, rows, dlogits): out fp32 [5] on the device, the batch means named by L.DISTILL_OUTPUTS
  (distance, the entropies of student and teacher, their task losses against `labels`, 0 without labels),
  summed in a fixed order; rows [5, n], the same per example; dlogits [n, dlogits_cols or C] =
  d distance / d student, zero in the columns past C.  Passing `dlogits` (a previous teacher's) adds to it."""
  _logits2d(student, teacher, labels, dlogits)
  if kind not in L.DIST_KINDS:
    raise ValueError(f"Unknown kind of distance {kind}.")
  n, C = student.shape
  assert teacher.shape == student.shape and (labels is None or labels.shape == student.shape)
  accumulate = dlogits is not None
  if want_grad and dlogits is None:
    dlogits = torch.empty((n, dlogits_cols or C), dtype=torch.float32, device=student.device)
  out = torch.empty(len(L.DISTILL_OUTPUTS), dtype=torch.float32, device=student.device)
  rows = torch.empty((len(L.DISTILL_OUTPUTS), n), dtype=torch.float32, device=student.device)
  L.call("bv_distill_loss", _p(student), student.stride(0), _p(teacher), teacher.stride(0), _p(labels),
         labels.stride(0) if labels is not None else 0, L.DIST_KINDS[kind], float(t), float(ls), int(accumulate),
         _p(dlogits), dlogits.stride(0) if dlogits is not None else 0, _p(out), _p(rows), n, C, _stream())
  return out, rows, dlogits


def distance(student, teacher, kind, epsilon=1e-12, t=1.0, ls=0.0, k=1):
  """dist() of evaluators/proj/distill/distance.py per row of student / teacher [n, C]: fp32 [n], int32 [n]
  for `agree`."""
  _logits2d(student, teacher)
  if kind not in L.DIST_KINDS:
    raise ValueError(f"Unknown kind of distance {kind}.")
  n, C = student.shape
  assert teacher.shape == student.shape
  out = torch.empty(n, dtype=torch.int32 if kind == "agree" else torch.float32, device=student.device)
  L.call("bv_distance", _p(student), student.stride(0), _p(teacher), teacher.stride(0), L.DIST_KINDS[kind],
         float(epsilon), float(t), float(ls), int(k), _p(out), n, C, _stream())
  return out


# ---- FlexiViT resampling (include/bv_b200_flexi.h) ----------------------------------------------------
def _resample_args(M, a):
  for t in (M, a):
    if t.dtype != torch.float32 or not t.is_contiguous():
      raise L.BvError(f"resampling takes contiguous fp32 matrices, got {t.dtype} {tuple(t.shape)} {t.stride()}")
  if M.dim() != 2 or a.dim() != 2:
    raise L.BvError(f"resampling takes a 2-D matrix and a 2-D operand, got {tuple(M.shape)} and {tuple(a.shape)}")
  return M.shape[0], M.shape[1], a.shape[1]


def resample_fwd(M, x, out=None):
  """M fp32 [R, K], x fp32 [K, J] -> bf16 [R, J] = M x (fp32 sums in ascending k, one rounding).  `out`: a
  contiguous bf16 buffer whose first R * J elements receive the result (e.g. a [Kp, d] GEMM operand)."""
  R, K, J = _resample_args(M, x)
  assert x.shape[0] == K, (tuple(M.shape), tuple(x.shape))
  if out is None:
    out = torch.empty((R, J), dtype=torch.bfloat16, device=x.device)
  assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.numel() >= R * J
  L.call("bv_resample_fwd", _p(M), _p(x), _p(out), R, K, J, _stream())
  return out


def resample_bwd(M, dy, dx):
  """dx fp32 [K, J] += M^T dy for M fp32 [R, K], dy fp32 [R, J] (fp32 sums in ascending r)."""
  R, K, J = _resample_args(M, dy)
  assert dy.shape[0] == R and dx.dtype == torch.float32 and dx.is_contiguous() and tuple(dx.shape) == (K, J), \
      (tuple(M.shape), tuple(dy.shape), tuple(dx.shape))
  L.call("bv_resample_bwd", _p(M), _p(dy), _p(dx), R, K, J, _stream())
  return dx


# ---- Jet normalizing flow (include/bv_b200_jet.h) -------------------------------------------------------
def _jet_args(*ts):
  for t in ts:
    if t is not None and (t.dtype not in (torch.float32, torch.bfloat16, torch.int32) or not t.is_contiguous()):
      raise L.BvError(f"Jet kernels take contiguous fp32 / bf16 / int32 buffers, got {t.dtype} {tuple(t.shape)}")


def jet_dequantize_patchify(image, ps, seed=0, counter=0, offset=0, noise_scale=1.0 / 127.5, out=None):
  """image fp32 [n, H, W, C] -> z fp32 [n, T, ps*ps*C] = patchified image + (uniform noise of the global
  Philox stream at element `offset` on) * noise_scale; noise_scale 0 is a plain patchify."""
  _jet_args(image, out)
  n, H, W, C = image.shape
  assert image.dtype == torch.float32
  if out is None:
    out = torch.empty((n, (H // ps) * (W // ps), ps * ps * C), dtype=torch.float32, device=image.device)
  L.call("bv_jet_dequantize_patchify", _p(image), _p(out), n, H, W, C, ps, int(seed), int(counter), int(offset),
         float(noise_scale), _stream())
  return out


def jet_unpatchify(z, image_shape, ps, out=None):
  """z fp32 [n, T, ps*ps*C] -> fp32 [n, H, W, C] (`image_shape`)."""
  _jet_args(z, out)
  n, H, W, C = image_shape
  if out is None:
    out = torch.empty((n, H, W, C), dtype=torch.float32, device=z.device)
  L.call("bv_jet_unpatchify", _p(z), _p(out), n, H, W, C, ps, _stream())
  return out


def jet_split(x, idx, T, c, out=None):
  """x fp32 [n, D] (any shape with n * D elements), idx int32 [D] -> x1 bf16 [n * T, c] = bf16(x[:, idx[:D/2]])."""
  _jet_args(x, idx, out)
  n = x.numel() // (2 * T * c)
  if out is None:
    out = torch.empty((n * T, c), dtype=torch.bfloat16, device=x.device)
  L.call("bv_jet_split", _p(x), _p(idx), _p(out), n, T, c, _stream())
  return out


def jet_coupling_fwd(x, idx, br, logdet, T, c, scale_factor=2.0, inverse=False, out=None):
  """One affine coupling (forward or inverse) of x fp32 [n, D] with br fp32 [n * T, 2c]; adds +-logdet of each
  image to logdet fp32 [n].  `out` may be x (in place).  Returns out."""
  _jet_args(x, idx, br, logdet, out)
  n = x.numel() // (2 * T * c)
  out = torch.empty_like(x) if out is None else out
  L.call("bv_jet_coupling_fwd", _p(x), _p(idx), _p(br), _p(out), _p(logdet), n, T, c, float(scale_factor),
         int(bool(inverse)), _stream())
  return out


def jet_coupling_bwd(dy, x, idx, br, dlogdet, T, c, scale_factor=2.0, dx=None, dbr=None):
  """Backward of jet_coupling_fwd: -> (dx, dbr).  dx fp32 like x receives d x2 (positions idx[D/2:]; `dx` may be
  dy), dbr bf16 [n * T, 2c] the gradient of br."""
  _jet_args(dy, x, idx, br, dx, dbr)
  n = x.numel() // (2 * T * c)
  dx = torch.empty_like(x) if dx is None else dx
  if dbr is None:
    dbr = torch.empty((n * T, 2 * c), dtype=torch.bfloat16, device=x.device)
  L.call("bv_jet_coupling_bwd", _p(dy), _p(x), _p(idx), _p(br), float(dlogdet), _p(dx), _p(dbr), n, T, c,
         float(scale_factor), _stream())
  return dx, dbr


def jet_merge_grad(dy, dx1, idx, T, c, dx=None):
  """dx[:, idx[:D/2]] = dy[:, idx[:D/2]] + dx1 (fp32 [n * T, c]); `dx` may be dy.  Returns dx."""
  _jet_args(dy, dx1, idx, dx)
  n = dy.numel() // (2 * T * c)
  dx = torch.empty_like(dy) if dx is None else dx
  L.call("bv_jet_merge_grad", _p(dy), _p(dx1), _p(idx), _p(dx), n, T, c, _stream())
  return dx


def jet_bits(z, logdet, grad_scale=None, dz=None):
  """z fp32 [n, ...], logdet fp32 [n] -> (rows fp32 [3, n], means fp32 [3]): bits, nll, logdet per dimension
  (each / (D ln 2)).  With grad_scale, dz (fp32 like z, allocated when None) = grad_scale * z; returns
  (rows, means, dz)."""
  _jet_args(z, logdet, dz)
  n = z.shape[0]
  D = z.numel() // n
  rows = torch.empty((3, n), dtype=torch.float32, device=z.device)
  means = torch.empty(3, dtype=torch.float32, device=z.device)
  if grad_scale is not None and dz is None:
    dz = torch.empty_like(z)
  L.call("bv_jet_bits", _p(z), _p(logdet), _p(rows), _p(means), _p(dz) if grad_scale is not None else None,
         float(grad_scale or 0.0), n, D, _stream())
  return (rows, means, dz) if grad_scale is not None else (rows, means)


# ---- integer evaluation paths -------------------------------------------------------------------
def top1(logits, labels=None, mask=None, want_idx=True):
  """argmax over classes (+ label gather and masked counts).  Returns (idx int32 [rows] or None,
  top1_correct fp32 [rows] or None, sums fp32 [2] = (ncorrect, nseen) or None)."""
  if not logits.is_cuda:
    raise L.BvError("bv_top1 needs CUDA tensors")
  logits, ld = _rowmajor(logits)
  rows, C = logits.shape
  idx = torch.empty(rows, dtype=torch.int32, device=logits.device) if want_idx else None
  correct = sums = None
  ldl = 0
  if labels is not None:
    labels, ldl = _rowmajor(labels.float())
    correct = torch.empty(rows, dtype=torch.float32, device=logits.device)
    sums = torch.zeros(2, dtype=torch.float32, device=logits.device)
    if mask is not None:
      mask = mask.float().contiguous()
  L.call("bv_top1", _p(logits), _dt(logits), rows, C, ld, _p(idx), _p(labels), ldl, _p(mask),
         _p(correct), _p(sums), _stream())
  return idx, correct, sums


def retrieval_ranks(dist, corr, t2i=True, i2t=True):
  """Positions of the positives in the ascending (stable) order of the columns / rows of the
  distance matrix dist [NI, NT] fp32; corr int32 [NT].  Returns (rank_t2i [NT], rank_i2t [NI])."""
  if not dist.is_cuda:
    raise L.BvError("bv_retrieval_ranks needs CUDA tensors")
  dist, ld = _rowmajor(dist)
  NI, NT = dist.shape
  corr = corr.to(device=dist.device, dtype=torch.int32).contiguous()
  r_t2i = torch.empty(NT, dtype=torch.int32, device=dist.device) if t2i else None
  r_i2t = torch.empty(NI, dtype=torch.int32, device=dist.device) if i2t else None
  L.call("bv_retrieval_ranks", _p(dist), NI, NT, ld, _p(corr), _p(r_t2i), _p(r_i2t), _stream())
  return r_t2i, r_i2t


# ---------------------------------------------------------------------------------------------------------
# BiT ResNet-v2 (include/bv_conv.h): NHWC bf16 activations, HWIO kernels.

def conv_out_size(h, k, stride):
  """Output size of the reference's k x k convolution with symmetric padding k // 2."""
  return (h + 2 * (k // 2) - k) // stride + 1


def _contig(*ts):
  for t in ts:
    if t is not None:
      assert t.is_contiguous(), "convolution operands must be contiguous"


def _conv_args(n, h, w, cin, cout, k, stride, **ptrs):
  a = L.ConvArgs(n=n, h=h, w=w, cin=cin, cout=cout, k=k, stride=stride)
  for name, t in ptrs.items():
    setattr(a, name, _p(t))
  return a


def conv_fwd(x, kernel, stride=1, resid=None):
  """y = conv(x, kernel) (+ resid): x bf16 [n, h, w, cin], kernel bf16 [k, k, cin, cout] (the standardised
  kernel).  Returns bf16 [n, ho, wo, cout].  A 1 x 1 stride-1 convolution is bv_gemm on [n h w, cin]; every
  other one is bv_conv_fwd."""
  n, h, w, cin = x.shape
  k, _, _, cout = kernel.shape
  _contig(x, kernel, resid)
  if k == 1 and stride == 1:     # a plain GEMM on [n h w, cin]
    aux = None if resid is None else resid.view(-1, cout)
    y = gemm(x.view(-1, cin), kernel.view(cin, cout), b_mn=True, aux=aux,
             epilogue=L.EPI_NONE if resid is None else L.EPI_BIAS_RESID)
    return y.view(n, h, w, cout)
  y = torch.empty((n, conv_out_size(h, k, stride), conv_out_size(w, k, stride), cout), dtype=torch.bfloat16,
                  device=x.device)
  a = _conv_args(n, h, w, cin, cout, k, stride, x=x, kernel=kernel, y=y, resid=resid)
  L.call("bv_conv_fwd", ctypes.byref(a), _stream())
  return y


def conv_dgrad(dy, kernel, h, w, stride=1, resid=None):
  """The input gradient [n, h, w, cin] (bf16) of conv_fwd for output gradient dy (+ resid)."""
  n, _, _, cout = dy.shape
  k, _, cin, _ = kernel.shape
  _contig(dy, kernel, resid)
  if k == 1 and stride == 1:
    aux = None if resid is None else resid.view(-1, cin)
    dx = gemm(dy.view(-1, cout), kernel.view(cin, cout), aux=aux,
              epilogue=L.EPI_NONE if resid is None else L.EPI_BIAS_RESID)
    return dx.view(n, h, w, cin)
  dx = torch.empty((n, h, w, cin), dtype=torch.bfloat16, device=dy.device)
  ws = torch.empty_like(dx) if stride == 2 else None
  a = _conv_args(n, h, w, cin, cout, k, stride, dy=dy, kernel=kernel, dx=dx, resid=resid, workspace=ws)
  L.call("bv_conv_dgrad", ctypes.byref(a), _stream())
  return dx


def conv_wgrad(x, dy, k, stride=1, out=None):
  """The kernel gradient fp32 [k, k, cin, cout] of conv_fwd; added into `out` when given."""
  n, h, w, cin = x.shape
  cout = dy.shape[-1]
  _contig(x, dy, out)
  acc = out is not None
  if k == 1 and stride == 1:
    dk = gemm(x.view(-1, cin), dy.view(-1, cout), a_mn=True, b_mn=True, out_dtype=torch.float32, reduce_out=True,
              out=None if out is None else out.view(cin, cout))
    return dk.view(1, 1, cin, cout)
  out = torch.empty((k, k, cin, cout), dtype=torch.float32, device=x.device) if out is None else out
  a = _conv_args(n, h, w, cin, cout, k, stride, x=x, dy=dy, dkernel=out)
  a.accumulate = int(acc)
  L.call("bv_conv_wgrad", ctypes.byref(a), _stream())
  return out


def weight_std_fwd(kernel):
  """bit_paper.standardize of an fp32 HWIO kernel: (bf16 standardised kernel, mean [cout], rstd [cout])."""
  _contig(kernel)
  cout = kernel.shape[-1]
  rows = kernel.numel() // cout
  ws = torch.empty(kernel.shape, dtype=torch.bfloat16, device=kernel.device)
  mean = torch.empty(cout, dtype=torch.float32, device=kernel.device)
  rstd = torch.empty_like(mean)
  L.call("bv_weight_std_fwd", _p(kernel), rows, cout, _p(ws), _p(mean), _p(rstd), _stream())
  return ws, mean, rstd


def weight_std_bwd(kernel, mean, rstd, g):
  """fp32 gradient of the kernel from g, the fp32 gradient of its standardised copy."""
  _contig(kernel, g)
  cout = kernel.shape[-1]
  dw = torch.empty_like(kernel)
  L.call("bv_weight_std_bwd", _p(kernel), _p(mean), _p(rstd), _p(g), kernel.numel() // cout, cout, _p(dw),
         _stream())
  return dw


def groupnorm_fwd(x, scale, bias, relu=True):
  """bit_paper.GroupNorm (32 groups) and an optional ReLU on bf16 NHWC x; returns (y, mean, rstd), the
  statistics fp32 [n, 32]."""
  _contig(x)
  n, c = x.shape[0], x.shape[-1]
  y = torch.empty_like(x)
  mean = torch.empty((n, 32), dtype=torch.float32, device=x.device)
  rstd = torch.empty_like(mean)
  L.call("bv_groupnorm_fwd", _p(x), _p(scale), _p(bias), _p(y), _p(mean), _p(rstd), n, x.numel() // (n * c), c,
         int(relu), _stream())
  return y, mean, rstd


def groupnorm_bwd(dy, x, scale, bias, mean, rstd, dscale, dbias, relu=True, dx_add=None):
  """dx (bf16, + dx_add when given) of groupnorm_fwd; dscale and dbias (fp32 [c]) are added into."""
  _contig(dy, x, dx_add)
  n, c = x.shape[0], x.shape[-1]
  dx = torch.empty_like(x)
  L.call("bv_groupnorm_bwd", _p(x), _p(dy), _p(scale), _p(bias), _p(mean), _p(rstd), _p(dx_add), _p(dx),
         _p(dscale), _p(dbias), n, x.numel() // (n * c), c, int(relu), _stream())
  return dx


def maxpool_fwd(x):
  """3 x 3 / 2 max pool with -inf padding (1, 1) of bf16 NHWC x."""
  _contig(x)
  n, h, w, c = x.shape
  y = torch.empty((n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), dtype=torch.bfloat16, device=x.device)
  L.call("bv_maxpool_fwd", _p(x), _p(y), n, h, w, c, _stream())
  return y


def maxpool_bwd(dy, x):
  _contig(dy, x)
  n, h, w, c = x.shape
  dx = torch.empty_like(x)
  L.call("bv_maxpool_bwd", _p(x), _p(dy), _p(dx), n, h, w, c, _stream())
  return dx


def stem_im2col(image):
  """The root convolution's 7 x 7 / 2 patches of an fp32 NHWC image [n, h, w, 3]: bf16
  [n * ho * wo, STEM_K_PAD] (columns past STEM_K are zero)."""
  _contig(image)
  n, h, w, _ = image.shape
  ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
  cols = torch.empty((n * ho * wo, L.STEM_K_PAD), dtype=torch.bfloat16, device=image.device)
  L.call("bv_stem_im2col", _p(image), _p(cols), n, h, w, _stream())
  return cols


def stem_conv_fwd(image, kernel):
  """The root block's 7 x 7 / 2 convolution (padding 3) of an fp32 image with the bf16 standardised kernel
  [7, 7, 3, cout]: bv_stem_im2col, then one GEMM with K = 147.  Returns bf16 [n, ho, wo, cout]."""
  n, h, w, _ = image.shape
  cout = kernel.shape[-1]
  cols = stem_im2col(image)
  y = gemm(cols[:, :L.STEM_K], kernel.reshape(L.STEM_K, cout), b_mn=True)
  return y.view(n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, cout)


def stem_conv_wgrad(image, dy):
  """fp32 [7, 7, 3, cout] kernel gradient of stem_conv_fwd (the patches are extracted again)."""
  cout = dy.shape[-1]
  cols = stem_im2col(image)
  dk = gemm(cols[:, :L.STEM_K], dy.reshape(-1, cout), a_mn=True, b_mn=True, out_dtype=torch.float32,
            reduce_out=True)
  return dk.view(7, 7, 3, cout)
