from openea_b200.models.trans.transe import TransE
from openea_b200.models.trans.transh import TransH
from openea_b200.models.trans.transd import TransD
from openea_b200.models.trans.transr import TransR
