"""Small helpers with the reference's names (modules/utils/util.py): task_divide :16, merge_dic :12,
generate_out_folder :33, load_session :6 (returns the engine's device session instead of a tf.Session)."""
import time


class EngineSession:
    """Stand-in for tf.Session: names the CUDA device the model's tables live on."""

    def __init__(self):
        import torch
        from openea_b200 import lib
        if not torch.cuda.is_available():
            raise lib.OeaError("the CUDA engine needs a CUDA device; there is no CPU fallback")
        lib.load()
        self.device = torch.device("cuda", torch.cuda.current_device())

    def close(self):
        pass


def load_session():
    return EngineSession()


def merge_dic(dic1, dic2):
    merged = dict(dic1)
    merged.update(dic2)
    return merged


def task_divide(idx, n):
    """Split `idx` into n contiguous chunks of ⌊len/n⌋ items, the last chunk taking the remainder; degenerate
    inputs (n <= 0, empty, n > len) come back as a single chunk and n == len as singletons."""
    total = len(idx)
    if n <= 0 or total == 0 or n > total:
        return [idx]
    if n == total:
        return [[item] for item in idx]
    size = total // n
    chunks = [idx[c * size:(c + 1) * size] for c in range(n - 1)]
    chunks.append(idx[(n - 1) * size:])
    return chunks


def generate_out_folder(out_folder, training_data_path, div_path, method_name):
    params = training_data_path.strip("/").split("/")
    print(out_folder, training_data_path, params, div_path, method_name)
    folder = "%s%s/%s/%s%s/" % (out_folder, method_name, params[-1], div_path, time.strftime("%Y%m%d%H%M%S"))
    print("results output folder:", folder)
    return folder
