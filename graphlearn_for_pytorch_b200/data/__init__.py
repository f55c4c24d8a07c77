from .graph import Topology, Graph
from .unified_tensor import UnifiedTensor
from .feature import DeviceGroup, Feature
from .reorder import sort_by_in_degree
from .dataset import Dataset, random_split
from .table_dataset import TableDataset
from . import vineyard_utils
from .vineyard_utils import (vineyard_to_csr, load_vertex_feature_from_vineyard, load_edge_feature_from_vineyard,
                             get_fid_from_gid, get_frag_vertex_offset, get_frag_vertex_num, VineyardPartitionBook,
                             VineyardGid2Lid, v6d_id_select, v6d_id_filter, write_arrow_fragments,
                             register_fragment_backend)
from .quantize import quantize_mxfp8, quantize_mxfp8_chunked, dequantize_mxfp8, mxfp8_row_bytes
# names the reference's `data` namespace re-exports from its helpers (python/data/__init__.py star imports)
from ..partition.partition_book import PartitionBook
from ..utils import convert_to_tensor, coo_to_csc, coo_to_csr, ptr2ind, share_memory, squeeze
from .dataset import rebuild_dataset, reduce_dataset
from .feature import rebuild_feature, reduce_feature
from .graph import rebuild_graph, reduce_graph
from .table_dataset import rebuild_table_dataset, reduce_table_dataset


def __getattr__(name):
  # `pywrap`: the native-module handle of the reference's Python layer (`from .. import py_graphlearn_torch as
  # pywrap`); resolved on first use because the facade imports this sub-package
  if name == 'pywrap':
    import importlib
    return importlib.import_module('..py_graphlearn_torch', __name__)
  raise AttributeError(name)
