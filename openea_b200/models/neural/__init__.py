from openea_b200.models._stubs import out_of_scope
from openea_b200.models.neural.proje import ProjE

ConvE = out_of_scope("ConvE", "2-D convolution scorer")
