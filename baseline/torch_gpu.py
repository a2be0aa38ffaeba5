"""LABELLED STAND-IN for the reference's JAX/XLA-GPU build (BASELINE.md section 2-A).

JAX / flax cannot be installed here or on the GPU box (no network, `import jax` fails on both), so
the "reference on the same GPU" number the north star asks for cannot be produced.  This file is
what BASELINE.md prescribes instead: the same models and the same update (forward, loss, backward,
gradient all-reduce, clip + Adam + decoupled weight decay) written in plain PyTorch -- bf16 autocast,
cuBLAS GEMMs, `scaled_dot_product_attention` (flash / cuDNN SDPA), fused Adam, DDP's bucketed
all-reduce -- i.e. the library-kernel implementation a practitioner would run on this box.  It is NOT
the reference and none of this repository's kernels, models or engine are on its path; `bench.py
--impl torch_gpu` times it on the same synthetic batch as the product arm.  That it computes the same
function is tested on CPU in float64 against the oracle (tests/test_oracle.py:
test_gpu_standin_computes_the_oracles_siglip_function, test_mixer_oracle_agrees_with_the_module_style_restatement).

Architectures restate big_vision/models/vit.py:57-281, models/proj/image_text/text_transformer.py:29-99,
models/proj/image_text/two_towers.py:28-90, models/mlp_mixer.py:30-124 and the loss of
trainers/proj/image_text/siglip.py:287-308 / utils.py:236-243,276-281.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.utils.checkpoint import checkpoint

VIT = {"S": (384, 12, 1536, 6), "B": (768, 12, 3072, 12), "L": (1024, 24, 4096, 16),
       "So400m": (1152, 27, 4304, 16), "G": (1664, 48, 8192, 16),
       "e": (1792, 56, 15360, 16)}
MIXER = {"B": (768, 12, 384, 3072)}


class Mlp(nn.Module):
  def __init__(self, d, m):
    super().__init__()
    self.fc1, self.fc2 = nn.Linear(d, m), nn.Linear(m, d)

  def forward(self, x):
    return self.fc2(F.gelu(self.fc1(x), approximate="tanh"))


class Attention(nn.Module):
  def __init__(self, d, heads):
    super().__init__()
    self.heads = heads
    self.q, self.kv, self.out = nn.Linear(d, d), nn.Linear(d, 2 * d), nn.Linear(d, d)

  def forward(self, xq, xkv):
    n, Nq, d = xq.shape
    h = self.heads
    q = self.q(xq).view(n, Nq, h, d // h).transpose(1, 2)
    k, v = self.kv(xkv).view(n, xkv.shape[1], 2, h, d // h).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(q, k, v)
    return self.out(o.transpose(1, 2).reshape(n, Nq, d))


class SelfAttention(nn.Module):
  def __init__(self, d, heads):
    super().__init__()
    self.heads = heads
    self.qkv, self.out = nn.Linear(d, 3 * d), nn.Linear(d, d)

  def forward(self, x):
    n, N, d = x.shape
    h = self.heads
    q, k, v = self.qkv(x).view(n, N, 3, h, d // h).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(q, k, v)
    return self.out(o.transpose(1, 2).reshape(n, N, d))


class Block(nn.Module):
  def __init__(self, d, m, heads):
    super().__init__()
    self.ln1, self.ln2 = nn.LayerNorm(d, eps=1e-6), nn.LayerNorm(d, eps=1e-6)
    self.attn, self.mlp = SelfAttention(d, heads), Mlp(d, m)

  def forward(self, x):
    x = x + self.attn(self.ln1(x))
    return x + self.mlp(self.ln2(x))


class Encoder(nn.Module):
  def __init__(self, d, depth, m, heads, remat=False):
    super().__init__()
    self.blocks = nn.ModuleList([Block(d, m, heads) for _ in range(depth)])
    self.norm = nn.LayerNorm(d, eps=1e-6)
    self.remat = remat

  def forward(self, x):
    for b in self.blocks:
      x = checkpoint(b, x, use_reentrant=False) if self.remat else b(x)
    return self.norm(x)


class ViT(nn.Module):
  def __init__(self, variant, res, num_classes=None, pool="gap", rep=False, remat=False):
    super().__init__()
    size, patch = variant.split("/")
    d, depth, m, heads = VIT[size]
    patch = int(patch)
    self.embed = nn.Conv2d(3, d, patch, patch)
    N = (res // patch) ** 2
    self.pos = nn.Parameter(torch.randn(1, N, d) / math.sqrt(d))
    self.cls = nn.Parameter(torch.zeros(1, 1, d)) if pool == "tok" else None
    self.encoder = Encoder(d, depth, m, heads, remat)
    self.pool = pool
    if pool == "map":
      self.probe = nn.Parameter(torch.randn(1, 1, d) * 0.02)
      self.map_attn, self.map_ln, self.map_mlp = Attention(d, heads), nn.LayerNorm(d, eps=1e-6), Mlp(d, m)
    self.rep = nn.Linear(d, d) if rep else None
    self.head = nn.Linear(d, num_classes) if num_classes else None

  def forward(self, image):                       # image: [n, H, W, 3] fp32 NHWC
    x = self.embed(image.permute(0, 3, 1, 2))      # NCHW view of the NHWC buffer (channels_last)
    x = x.flatten(2).transpose(1, 2) + self.pos.to(x.dtype)
    if self.cls is not None:
      x = torch.cat([self.cls.to(x.dtype).expand(x.shape[0], -1, -1), x], 1)
    x = self.encoder(x)
    if self.pool == "map":
      y = self.map_attn(self.probe.to(x.dtype).expand(x.shape[0], -1, -1), x)
      x = (y + self.map_mlp(self.map_ln(y)))[:, 0]
    elif self.pool == "gap":
      x = x.mean(1)
    else:
      x = x[:, 0]
    if self.rep is not None:
      x = torch.tanh(self.rep(x))
    return self.head(x) if self.head is not None else x


class TextTower(nn.Module):
  def __init__(self, size, vocab, length, out, remat=False):
    super().__init__()
    d, depth, m, heads = VIT[size]
    self.embed = nn.Embedding(vocab, d)
    self.pos = nn.Parameter(torch.randn(1, length, d) / math.sqrt(d))
    self.encoder = Encoder(d, depth, m, heads, remat)
    self.head = nn.Linear(d, out)

  def forward(self, ids):
    x = self.embed(ids.long()) + self.pos
    return self.head(self.encoder(x)[:, -1])


class TwoTowers(nn.Module):
  def __init__(self, img_variant, txt_size, res, out, remat=False, freeze_img=False):
    super().__init__()
    self.img = ViT(img_variant, res, None, pool="map", remat=remat)
    self.txt = TextTower(txt_size, 32_000, 64, out, remat)
    self.t = nn.Parameter(torch.tensor([math.log(10.0)]))
    self.b = nn.Parameter(torch.tensor([-10.0]))
    # locked-image tuning (SigLiT): the image tower gets no gradient and its forward records no graph
    self.freeze_img = freeze_img
    if freeze_img:
      self.img.requires_grad_(False)

  def forward(self, image, text):
    if self.freeze_img:
      with torch.no_grad():
        zi = self.img(image).float()
    else:
      zi = self.img(image).float()
    zt = self.txt(text).float()
    zi = zi / (zi.norm(dim=-1, keepdim=True) + 1e-8)
    zt = zt / (zt.norm(dim=-1, keepdim=True) + 1e-8)
    return zi, zt


class MixerBlock(nn.Module):
  def __init__(self, d, N, tok, ch):
    super().__init__()
    self.ln1, self.ln2 = nn.LayerNorm(d, eps=1e-6), nn.LayerNorm(d, eps=1e-6)
    self.tok, self.ch = Mlp(N, tok), Mlp(d, ch)

  def forward(self, x):
    x = x + self.tok(self.ln1(x).transpose(1, 2)).transpose(1, 2)
    return x + self.ch(self.ln2(x))


class Mixer(nn.Module):
  def __init__(self, variant, res, num_classes):
    super().__init__()
    size, patch = variant.split("/")
    d, blocks, tok, ch = MIXER[size]
    patch = int(patch)
    self.stem = nn.Conv2d(3, d, patch, patch)
    N = (res // patch) ** 2
    self.blocks = nn.ModuleList([MixerBlock(d, N, tok, ch) for _ in range(blocks)])
    self.norm = nn.LayerNorm(d, eps=1e-6)
    self.head = nn.Linear(d, num_classes)

  def forward(self, image):
    x = self.stem(image.permute(0, 3, 1, 2)).flatten(2).transpose(1, 2)
    for b in self.blocks:
      x = b(x)
    return self.head(self.norm(x).mean(1))


def siglip_loss(zimg, ztxt_all, t, b, row_offset, global_b):
  logits = zimg @ ztxt_all.T * t.exp() + b
  n = zimg.shape[0]
  m = -torch.ones_like(logits)
  idx = torch.arange(n, device=logits.device)
  m[idx, row_offset + idx] = 1.0
  return -F.logsigmoid(m * logits).sum() / global_b


def make_step(workload, world, rank, device):
  """Returns (step_fn(batch) -> loss tensor, n_params).  `workload` is bench.py's registry entry."""
  import torch.distributed as dist
  kind = workload["kind"]
  if kind == "siglip":
    kw = workload["model_kw"]
    model = TwoTowers(kw["image"]["variant"], kw["text"]["variant"], workload["res"], kw["out_dim"][1],
                      remat=workload.get("remat", False), freeze_img=workload.get("freeze_img", False))
  elif workload["model"] == "vit":
    kw = workload["model_kw"]
    model = ViT(kw["variant"], workload["res"], workload["num_classes"], pool=kw.get("pool_type", "gap"),
                rep=bool(kw.get("rep_size")), remat=workload.get("remat", False))
  else:
    model = Mixer(workload["model_kw"]["variant"], workload["res"], workload["num_classes"])
  model = model.to(device).to(memory_format=torch.channels_last)
  # decoupled weight decay on the matmul / conv kernels only (optax.py:133 mask `.*/kernel$`)
  decay = [m.weight for m in model.modules() if isinstance(m, (nn.Linear, nn.Conv2d)) and m.weight.requires_grad]
  ids = {id(p) for p in decay}
  rest = [p for p in model.parameters() if id(p) not in ids and p.requires_grad]
  opt = torch.optim.AdamW([{"params": decay, "weight_decay": 1e-4}, {"params": rest, "weight_decay": 0.0}],
                          lr=1e-3, betas=(0.9, 0.95), fused=True)
  net = model
  if world > 1:
    net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[device.index], gradient_as_bucket_view=True)
  params = [p for p in model.parameters() if p.requires_grad]

  def step(batch):
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
      if kind == "siglip":
        zi, zt = net(batch["image"], batch["labels"])
      else:
        logits = net(batch["image"]).float()
    if kind == "siglip":
      n = zi.shape[0]
      if world > 1:
        import torch.distributed.nn.functional as dfn
        zt_all = torch.cat(dfn.all_gather(zt), 0)
      else:
        zt_all = zt
      # DDP averages gradients over ranks: scale the per-rank partial of the GLOBAL-batch loss by world
      loss = siglip_loss(zi, zt_all, model.t, model.b, rank * n, n * world) * world
    elif workload["loss"] == "sigmoid_xent":
      y = batch["labels"]
      loss = -(y * F.logsigmoid(logits) + (1 - y) * F.logsigmoid(-logits)).sum(-1).mean()
    else:
      loss = -(batch["labels"] * F.log_softmax(logits, -1)).sum(-1).mean()
    loss.backward()
    torch.nn.utils.clip_grad_norm_(params, 1.0, foreach=True)
    opt.step()
    return loss.detach()

  return step, sum(p.numel() for p in params)
