from openea_b200.models.semantic.distmult import DistMult
from openea_b200.models.semantic.hole import HolE
from openea_b200.models.semantic.rotate import RotatE
from openea_b200.models.semantic.simple import SimplE
