from .sage import SAGEConv, GraphSAGE, GraphSageEngine
from .sage_link import GraphSageLinkEngine, link_auc
from .sage_multilabel import GraphSageMultiLabelEngine, multilabel_auc, multilabel_f1, pack_label_bits
from .trainer import GraphSageTrainer, GraphSageMultiLabelTrainer, GraphSageLinkTrainer
from .rgnn import RGNN, RelSAGEConv, RelGCNConv, RelGATConv
from .seal import drnl_node_labeling, DGCNN
from .hgt import HGT, HGTConv
from .hetero_engine import HeteroSageEngine
from .hetero_gat_engine import HeteroGatEngine
from .hetero_hgt_engine import HeteroHgtEngine
from .metapath2vec import MetaPath2VecEngine
from .seal_engine import SealEngine
from .label_prop import LabelPropagation, CorrectAndSmooth
from .link_rank import link_topk, link_scores, link_recall_at_k, link_hits_at_k, link_mrr
from .kge import KgeEngine, kge_filter
