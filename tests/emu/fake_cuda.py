"""TEST INFRASTRUCTURE: runs GPU-only Python entry points of this repository (bench.py, __graft_entry__.smoke) in a
process where torch's CUDA surface is faked and liboea's entry points are served by the CPU warp emulator, so that their
Python logic — argument plumbing, JSON contract, probe choreography — is exercised where no GPU exists.  Numbers printed
this way are meaningless as measurements.  Only tests/test_bench_on_emulator.py starts this, in a subprocess.

    python tests/emu/fake_cuda.py bench [bench.py arguments…]      (a `micro` workload is registered)
    python tests/emu/fake_cuda.py probe
    python tests/emu/fake_cuda.py smoke
    python tests/emu/fake_cuda.py lifecycle <Approach> <tmp folder>
    python tests/emu/fake_cuda.py pytest <pytest arguments…>      (ad-hoc: GPU-marked tests against the emulator)
"""
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import pytest  # noqa: E402
import torch  # noqa: E402

from openea_b200 import engine as eng  # noqa: E402
from openea_b200 import finding  # noqa: E402
from tests.emu import build_emu  # noqa: E402


def install():
    build_emu.patch_engine(pytest.MonkeyPatch(), build_emu.load())      # for the life of the process
    cpu = torch.device("cpu")

    class Stream:
        def __init__(self, *a, **k):
            self.cuda_stream = 0x10

        def synchronize(self):
            pass

    class Event:
        count = 0

        def __init__(self, *a, **k):
            Event.count += 1
            self.cuda_event, self.t = 0x100 + Event.count, None

        def record(self, *a, **k):
            self.t = time.perf_counter()

        def elapsed_time(self, other):
            return 1e3 * (other.t - self.t)

        def synchronize(self):
            pass
    torch.cuda.Stream, torch.cuda.Event = Stream, Event
    torch.cuda.synchronize = torch.cuda.set_device = lambda *a, **k: None
    torch.cuda.is_available = lambda: True
    torch.cuda.current_device = lambda: 0
    torch.Tensor.cuda = torch.Tensor.pin_memory = lambda self, *a, **k: self
    torch.Tensor.is_pinned = lambda self, *a, **k: True
    torch.Tensor.cpu = lambda self, *a, **k: self.clone()      # a device → host read is a copy, never an alias
    real_device = torch.device

    class _DeviceMeta(type):                # torch.device stays usable as a type (isinstance, `torch.device | None`)
        def __call__(cls, *a, **k):
            return real_device("cpu")

        def __instancecheck__(cls, obj):
            return isinstance(obj, real_device)

        def __or__(cls, other):
            return real_device | other

        def __ror__(cls, other):
            return other | real_device

    class CpuDevice(metaclass=_DeviceMeta):
        pass
    torch.device = CpuDevice
    finding._device = lambda: cpu
    table_init = eng.EmbeddingTable.__init__
    eng.EmbeddingTable.__init__ = lambda self, init, l2_norm, optimizer="Adagrad", device="cpu": table_init(
        self, init, l2_norm, optimizer, "cpu")
    trainer_init = eng.TripleTrainer.__init__

    def trainer(self, *a, **k):
        trainer_init(self, *a, **k)
        self._loss_pinned = torch.zeros(1, dtype=torch.float64)
    eng.TripleTrainer.__init__ = trainer

    def is_cuda_name(x):
        return (isinstance(x, str) and x.startswith("cuda")) or (isinstance(x, real_device) and x.type == "cuda")

    class CudaToCpu(torch.overrides.TorchFunctionMode):     # device="cuda" / .to("cuda") anywhere in torch's API → CPU
        def __torch_function__(self, func, types, args=(), kwargs=None):
            kwargs = dict(kwargs or {})
            if is_cuda_name(kwargs.get("device")):
                kwargs["device"] = "cpu"
            args = tuple("cpu" if is_cuda_name(a) else a for a in args)
            return func(*args, **kwargs)
    CudaToCpu().__enter__()

    class EagerEpoch:                      # CUDA graphs need a device: replay = the same steps, eagerly
        def __init__(self, tr, kg1, kg2, tset, batch, k, steps, max_try=10):
            self.args = (tr, kg1, kg2, tset, batch, k, steps)

        def replay(self, seed):
            tr, kg1, kg2, tset, batch, k, steps = self.args
            for step in range(steps):
                tr.step_sampled(kg1, kg2, tset, batch, k, step, seed)
    eng.EpochGraph = EagerEpoch

    # one process per "GPU" on the CPU: torch.distributed joins a gloo group whatever backend the caller names, so that the
    # N > 1 control flow of bench.py (exchange cadence, matched collectives, sharded CSLS) can run under the emulator
    import torch.distributed as dist
    real_init = dist.init_process_group

    def init_gloo(backend=None, *a, **k):
        k.pop("device_id", None)
        return real_init("gloo", *a, **k)
    dist.init_process_group = init_gloo


def lifecycle(name, folder):
    """set_args / set_kgs / init / run / test / save of one approach on the micro synthetic dataset, two epochs."""
    from openea_b200 import approaches, presets
    presets.gcn_align, presets.bootea_transh = presets.gcn_align, presets.bootea_transh      # preset names are lower-cased class names
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.synth import write_dataset
    data = write_dataset(os.path.join(folder, "micro") + "/", "micro")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:      # one process per "GPU": what run/main_from_args.py does under torchrun (gloo here, see install())
        import torch.distributed as dist
        dist.init_process_group("nccl", rank=int(os.environ["RANK"]), world_size=world)
    args = getattr(presets, name.lower())("15K")
    if os.environ.get("OEA_MULTI_MODE"):
        args.multi_gpu_mode = os.environ["OEA_MULTI_MODE"]
    args.training_data, args.output = data, os.path.join(folder, "out") + "/"
    args.batch_size, args.max_epoch, args.start_valid, args.eval_freq, args.dim, args.cuda_graph = 64, 2, 1, 1, 16, False
    # sizes that only make sense on real datasets (125 hard negatives, a 2 % candidate list) scaled to 40 entities
    for key, val in dict(bp_freq=1, sim_th=0.05, attr_max_epoch=2, sub_mat_size=4, attr_sim_mat_threshold=0.5,
                         truncated_epsilon=0.5).items():
        if hasattr(args, key):
            setattr(args, key, val)
    if hasattr(args, "neg_triple_num"):
        args.neg_triple_num = min(args.neg_triple_num, 3)
    from openea_b200.models import semantic, trans
    cls = next(getattr(m, name) for m in (approaches, trans, semantic) if hasattr(m, name))
    model = cls()
    model.set_args(args)
    model.set_kgs(read_kgs_from_folder(data, args.dataset_division, args.alignment_module, args.ordered))
    model.init()
    model.run()
    model.test()
    model.save()
    if world == 1 or int(os.environ["RANK"]) == 0:
        assert os.path.exists(model.out_folder + "ent_embeds.npy")
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
    print("lifecycle ok:", name)


def main():
    install()
    what, rest = sys.argv[1], sys.argv[2:]
    if what == "lifecycle":
        return lifecycle(rest[0], rest[1])
    if what == "pytest":                     # ad-hoc audits: GPU-marked tests executed against the emulator
        return pytest.main(rest)
    if what == "smoke":
        import __graft_entry__
        return __graft_entry__.smoke()
    import bench
    bench.WORKLOADS["micro"] = dict(shape="micro", dim=16, batch=48, k=3, eps=0.5, lr=0.01, margin=0.01, neg_margin=2.0,
                                    balance=0.2, name="micro (emulator)")
    bench.L2_FLUSH_BYTES = 1 << 20
    if what == "probe":
        return bench.probe_pipelined_e2e(types.SimpleNamespace(workload="micro", steps=8))
    sys.argv = ["bench.py"] + rest
    return bench.main()


if __name__ == "__main__":
    sys.exit(main() or 0)
