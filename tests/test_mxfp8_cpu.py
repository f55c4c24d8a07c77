"""MXFP8 feature storage on the host: the quantiser's row layout at every width the kernels accept, the chunked
quantiser, and the engines' format checks that need no device."""
from types import SimpleNamespace

import pytest
import torch

from graphlearn_for_pytorch_b200.data import (dequantize_mxfp8, mxfp8_row_bytes, quantize_mxfp8,
                                              quantize_mxfp8_chunked)
from graphlearn_for_pytorch_b200.models.hetero_engine import resolve_feature_formats

WIDTHS = [32, 64, 96, 128, 160, 256, 480, 512, 992, 1024]


@pytest.mark.parametrize('d', WIDTHS)
def test_row_layout_scales_padding_and_round_trip(d):
  nb = d // 32
  assert mxfp8_row_bytes(d) % 16 == 0 and d + nb <= mxfp8_row_bytes(d) < d + nb + 16
  g = torch.Generator().manual_seed(d)
  x = torch.randn(200, d, generator=g) * torch.exp2(torch.randint(-8, 9, (200, nb), generator=g).float()).repeat_interleave(32, 1)
  x[7] = 0                                   # an all-zero row
  x[9, 32 * (nb - 1):] = 0                   # an all-zero last block
  q = quantize_mxfp8(x)
  assert q.dtype == torch.uint8 and q.shape == (200, mxfp8_row_bytes(d))
  assert bool((q[:, d + nb:] == 0).all()), 'padding bytes are zero'
  # scale byte b of a block = 127 + the smallest exponent e with amax / 2^e <= 448; all-zero blocks carry e = -126
  amax = x.view(200, nb, 32).abs().amax(2)
  e = q[:, d:d + nb].float() - 127
  live = amax > 0
  assert bool((amax[live] / torch.exp2(e[live]) <= 448).all()) and bool((amax[live] / torch.exp2(e[live] - 1) > 448).all())
  assert bool((e[~live] == -126).all()) and bool((q[:, d:d + nb] >= 1).all())
  y = dequantize_mxfp8(q, d)
  assert bool((y[7] == 0).all()) and bool((y[9, 32 * (nb - 1):] == 0).all())
  # e4m3 keeps 3 mantissa bits: relative error <= 2^-4 of the element, or half the smallest subnormal step of its block
  step = torch.exp2(e).repeat_interleave(32, 1) * 2.0 ** -9
  assert bool(((y - x).abs() <= x.abs() * 2.0 ** -4 + step / 2).all())
  # de-quantised values are bf16 values, and quantising them again loses nothing
  assert torch.equal(y.to(torch.bfloat16).float(), y)
  assert torch.equal(dequantize_mxfp8(quantize_mxfp8(y), d), y)


def test_chunked_quantiser_equals_the_one_shot_quantiser():
  x = torch.randn(1000, 96, generator=torch.Generator().manual_seed(0)).to(torch.bfloat16)
  ref = quantize_mxfp8(x)
  for rows in (1, 7, 333, 1000, 5000):
    assert torch.equal(quantize_mxfp8_chunked(x, rows), ref)


def _tbl(width, uint8):
  return SimpleNamespace(width=width, is_uint8=uint8)


def test_engine_format_checks():
  dims = {'paper': 1024, 'author': 256, 'inst': 72}
  tables = {'paper': _tbl(mxfp8_row_bytes(1024), True), 'author': _tbl(256, False), 'inst': _tbl(72, False)}
  assert resolve_feature_formats({'paper': 'mxfp8'}, dims, tables) == {'paper': 'mxfp8', 'author': 'bf16', 'inst': 'bf16'}
  assert resolve_feature_formats('bf16', dims, dict(tables, paper=_tbl(1024, False))) == dict.fromkeys(dims, 'bf16')
  with pytest.raises(ValueError, match='uint8 feature table'):
    resolve_feature_formats('bf16', dims, tables)
  with pytest.raises(ValueError, match='multiple of 32'):
    resolve_feature_formats({'inst': 'mxfp8'}, dims, dict(tables, paper=_tbl(1024, False)))   # inst: 72 columns
  with pytest.raises(ValueError, match='mxfp8_row_bytes'):
    resolve_feature_formats({'paper': 'mxfp8', 'author': 'mxfp8'}, dims, tables)   # author holds bf16 rows
  with pytest.raises(ValueError, match='mxfp8_row_bytes'):
    resolve_feature_formats({'paper': 'mxfp8'}, dims, dict(tables, paper=_tbl(1024 + 16, True)))
  with pytest.raises(ValueError, match="'bf16' or 'mxfp8'"):
    resolve_feature_formats({'paper': 'fp8'}, dims, tables)


def test_graphsage_engine_format_checks_need_no_device():
  from graphlearn_for_pytorch_b200.models import GraphSageEngine
  labels = torch.zeros(4, dtype=torch.int64)
  with pytest.raises(ValueError, match='multiple of 32'):
    GraphSageEngine(None, _tbl(96, True), labels, in_dim=72, num_nodes=4, feature_format='mxfp8')
  with pytest.raises(ValueError, match='mxfp8_row_bytes'):
    GraphSageEngine(None, _tbl(256 + 32, True), labels, in_dim=256, num_nodes=4, feature_format='mxfp8')
  with pytest.raises(ValueError, match='mxfp8_row_bytes'):
    GraphSageEngine(None, _tbl(128, False), labels, in_dim=128, num_nodes=4, feature_format='mxfp8')
