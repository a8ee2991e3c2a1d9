from openea_b200.approaches.aligne import AlignE
from openea_b200.approaches.attr2vec import Attr2Vec
from openea_b200.approaches.attre import AttrE
from openea_b200.approaches.bootea import BootEA
from openea_b200.approaches.bootea_rotate import BootEA_RotatE
from openea_b200.approaches.bootea_transh import BootEA_TransH
from openea_b200.approaches.imuse import IMUSE
from openea_b200.approaches.iptranse import IPTransE
from openea_b200.approaches.jape import JAPE
from openea_b200.approaches.mtranse import MTransE
from openea_b200.approaches.sea import SEA
from openea_b200.models._stubs import out_of_scope
from openea_b200.approaches.alinet import AliNet
from openea_b200.approaches.gcn_align import GCN_Align
from openea_b200.approaches.rdgcn import RDGCN

RSN4EA = out_of_scope("RSN4EA", "recurrent skipping network over paths")
MultiKE = out_of_scope("MultiKE", "multi-view literal/attribute encoders")
GMNN = out_of_scope("GMNN", "graph matching network")
KDCoE = out_of_scope("KDCoE", "description encoder co-training")
