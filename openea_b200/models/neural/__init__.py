from openea_b200.models.neural.conve import ConvE
from openea_b200.models.neural.proje import ProjE
