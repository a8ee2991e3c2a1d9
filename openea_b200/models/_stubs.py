"""Importable placeholders for reference classes that are OUT OF SCOPE of the CUDA hot path (SURVEY §2:
attribute/literal encoders, RNN paths, graph matching, FFT/conv/complex KGE models).  They keep
run/main_from_args.py importable; using one fails loudly instead of silently running something else."""
from openea_b200.models.basic_model import BasicModel


def out_of_scope(name, reason):
    def init(self):
        raise NotImplementedError("%s is outside the accelerated hot path of this engine (%s); "
                                  "use the reference implementation for it" % (name, reason))
    return type(name, (BasicModel,), {"init": init, "__doc__": "Out of scope: " + reason})
