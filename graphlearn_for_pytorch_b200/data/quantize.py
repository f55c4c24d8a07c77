"""MXFP8 feature storage (OCP microscaling format): e4m3 elements with one power-of-two UE8M0 scale per block of 32.

The reference stores features as fp32 / fp16 / bf16 tensors (python/data/feature.py; csrc/cuda/unified_tensor.cu:112-130
registers the dtypes).  The feature gather of layer 1 is bound by bytes moved (local HBM and, for partitioned
tables, NVLink), so halving the row size is worth more than any kernel tweak: a d-wide row becomes

    [ d bytes e4m3 | d/32 bytes UE8M0 scales | zero padding to a multiple of 16 bytes ]

(d = 128: 144 bytes instead of 256; d = 1024: 1056 instead of 2048).  The rows are de-quantised in registers by
every kernel that reads a feature table, at any d that is a multiple of 32 up to 1024 unless noted:

  k_sage_aggregate            layer-1 neighbour mean of the sampled batch (csrc/cuda/sage.cu): GraphSageEngine's
                              unfused layer 1 and the heterogeneous engines' per-relation column blocks
  k_sage_fused3               fused layer-1 gather + GEMM of GraphSageEngine (csrc/cuda/sage_tc.cu), d = 128 only
  k_gather_mxfp8_vec          `RowTableHandle.gather_mxfp8_into`: rows into a bf16 column block, device-side count
                              (the engines' self blocks and the attention engines' layer-1 inputs)
  k_gather_mxfp8              `RowTableHandle.gather_mxfp8`: a fresh dense bf16 [n, d], d a multiple of 128
  k_sage_full_aggregate       exact full-neighbourhood inference of every engine (csrc/cuda/sage_infer.cu)

Everything downstream still sees bf16 / fp32.
"""
import torch

BLOCK = 32
E4M3_MAX = 448.0


def mxfp8_row_bytes(d: int) -> int:
  return (d + d // BLOCK + 15) // 16 * 16


def quantize_mxfp8(x: torch.Tensor) -> torch.Tensor:
  """[N, d] float/bf16 (d a multiple of 32)  ->  uint8 [N, mxfp8_row_bytes(d)] packed rows."""
  assert x.dim() == 2 and x.shape[1] % BLOCK == 0
  n, d = x.shape
  xf = x.float().view(n, d // BLOCK, BLOCK)
  amax = xf.abs().amax(dim=2)
  # smallest power of two s with amax / s <= 448
  e = torch.ceil(torch.log2(torch.clamp(amax, min=1e-30) / E4M3_MAX)).clamp(-126, 127)
  e = torch.where(amax > 0, e, torch.full_like(e, -126))
  scale = torch.exp2(e).unsqueeze(2)
  q = (xf / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(n, d)
  out = torch.zeros(n, mxfp8_row_bytes(d), dtype=torch.uint8, device=x.device)
  out[:, :d] = q.view(torch.uint8)
  out[:, d:d + d // BLOCK] = (e + 127).to(torch.uint8)
  return out


def dequantize_mxfp8(rows: torch.Tensor, d: int) -> torch.Tensor:
  """Inverse of `quantize_mxfp8` (fp32 [N, d]); the reference semantics for the device de-quantisers."""
  n = rows.shape[0]
  q = rows[:, :d].contiguous().view(torch.float8_e4m3fn).float().view(n, d // BLOCK, BLOCK)
  e = rows[:, d:d + d // BLOCK].float() - 127.0
  return (q * torch.exp2(e).unsqueeze(2)).view(n, d)


def quantize_mxfp8_chunked(x: torch.Tensor, rows: int = 1 << 20) -> torch.Tensor:
  """`quantize_mxfp8(x)` computed `rows` rows at a time, so that the fp32 temporaries of the quantiser never cover the
  whole table (a 1024-wide table of 10^7 rows would need 40 GB of them)."""
  n = x.shape[0]
  if n <= rows:
    return quantize_mxfp8(x)
  return torch.cat([quantize_mxfp8(x[b0:min(n, b0 + rows)]) for b0 in range(0, n, rows)])
