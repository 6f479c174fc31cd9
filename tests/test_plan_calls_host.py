"""What the Python plan wrappers pass to the library, without a GPU: plans of every kind are created by the real library
with a NULL context, then the context's library is replaced by a recorder.  Every run and derivative entry (and the
all-reduce) is logged with its scalar arguments, array contents, null / non-null pointers and requested output slots, and
every upload, download, adoption and free of a DeviceTensor with its shape and contents.  Each public method of
NetworkPlan and SlicedPlan, with host inputs, must produce the log in CALLS."""
import ctypes as C
import types

import numpy as np
import pytest

from tnc_b200._lib import TncbPath, TncbTn

# metadata entries the recorder passes to the library: creation, layout and teardown
PASSTHROUGH = {"tncb_network_out_legs", "tncb_plan_grad_offsets", "tncb_plan_info", "tncb_plan_destroy", "tncb_last_error"}
# the trailing output arguments of each logged entry: "r" a tensor of the result's dims, "g" a gradient block, "c" a leading
# count, 0 the legs of a contracted result
OUT_SHAPES = {"tncb_plan_run": ["r", 0, 0], "tncb_plan_execute": ["r", 0, 0], "tncb_plan_run_slices": ["r", 0, 0],
              "tncb_plan_run_batch": ["cr", 0, 0],
              "tncb_plan_vjp": ["g"], "tncb_plan_vjp_sliced": ["r", "g"], "tncb_plan_vjp_batch": ["cr", "cg", "g"],
              "tncb_plan_jvp": ["r", "r"], "tncb_plan_jvp_sliced": ["r", "r"], "tncb_plan_jvp_batch": ["cr", "cr"],
              "tncb_plan_hvp": ["r", "r", "g", "g"], "tncb_plan_hvp_sliced": ["r", "r", "g", "g"],
              "tncb_plan_hvp_batch": ["cr", "cr", "cg", "g", "cg", "g"]}
COUNT_ARG = {"tncb_plan_run_batch": 3, "tncb_plan_vjp_batch": 3, "tncb_plan_jvp_batch": 3, "tncb_plan_hvp_batch": 2}


def network():
    """A(0, 1) B(1, 2) C(2, 3), leaf dims 2 x 3, 3 x 2, 2 x 2, small integer payloads: the result has legs [3, 0]"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(7)
    parts = []
    for legs, dims in (([0, 1], [2, 3]), ([1, 2], [3, 2]), ([2, 3], [2, 2])):
        t = Tensor(legs, dims)
        t.set_tensor_data(TensorData.Matrix(rng.integers(-3, 4, dims) + 1j * rng.integers(-3, 4, dims)))
        parts.append(t)
    return Tensor.new_composite(parts), ContractionPath.simple([(0, 1), (0, 2)])


class Recorder:
    """Stands in for the library of a context: logged entries write dummy handles into the requested outputs"""

    def __init__(self, lib, log, names, result):
        self._lib, self._log, self._names, self._result = lib, log, names, result

    def __getattr__(self, name):
        if name in PASSTHROUGH or name.startswith("tncb_plan_create"):
            return getattr(self._lib, name)
        return lambda *args: self._call(name, args)

    def _call(self, name, args):
        legs, dims = self._result
        te = 2 * 3 + 3 * 2 + 2 * 2
        count = int(args[COUNT_ARG[name]]) if name in COUNT_ARG else None
        outs = OUT_SHAPES.get(name, [])
        kinds = [None] * (len(args) - len(outs)) + outs
        row = [name]
        for a, kind in list(zip(args, kinds))[1:]:
            row.append(self._describe(a, kind, count, legs, dims, te))
        self._log.append(tuple(row))
        return 0

    def _describe(self, a, kind, count, legs, dims, te):
        if a is None:
            return None
        if type(a).__name__ == "CArgObject":
            obj = a._obj
            if isinstance(obj, C.c_void_p):                # an output tensor slot
                shape = ((count,) if "c" in kind else ()) + (tuple(dims) if "r" in kind else (te,))
                tag = f"out{len(self._names)}"
                obj.value = 0x7000 + len(self._names)
                self._names[obj.value] = (tag, shape)
                return "out"
            if isinstance(obj, C.c_int):
                obj.value = len(legs)
                return "n_out"
            if isinstance(obj, TncbTn):
                return "node"
            if isinstance(obj, TncbPath):
                return "path"
            raise AssertionError(type(obj))
        if isinstance(a, C.Array):
            if a._type_ is C.c_uint64 and len(a) == 64 and not any(a):   # the result legs
                for i, l in enumerate(legs):
                    a[i] = l
                return "legs"
            if a._type_ is C.c_void_p:
                return ("ptrs", [None if p is None else "ptr" for p in a])
            if a._type_ is C.c_uint64:
                return ("u64", list(a))
            return ("nodes", len(a))
        if isinstance(a, C.c_void_p):
            return self._names.get(a.value, ("handle",))[0] if a.value else None
        if isinstance(a, int):
            return a
        raise AssertionError(type(a))


@pytest.fixture
def rec(built_lib, monkeypatch):
    """(plans by kind, the log): plans on a context whose library is a Recorder, DeviceTensor patched to log"""
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = network()
    log, names = [], {}
    ctx = types.SimpleNamespace(_l=built_lib, handle=None, device=0)
    plans = {"plain": NetworkPlan(tn, path, ctx=ctx), "vjp": NetworkPlan.for_gradients(tn, path, ctx=ctx),
             "jvp": NetworkPlan.for_tangents(tn, path, ctx=ctx), "hvp": NetworkPlan.for_hvp(tn, path, ctx=ctx),
             "sliced vjp": SlicedPlan.for_gradients(tn, path, [1], ctx=ctx),
             "sliced jvp": SlicedPlan.for_tangents(tn, path, [1], ctx=ctx),
             "sliced hvp": SlicedPlan.for_hvp(tn, path, [1], ctx=ctx)}
    ctx._l = Recorder(built_lib, log, names, ([3, 0], [2, 2]))
    plans["sliced"] = SlicedPlan(tn, path, [1], ctx=ctx)
    for p in plans.values():
        names[(p.plan if hasattr(p, "plan") else p).handle.value] = ("plan", None)

    def make(ctx, arr, kind):
        tag = f"up{len(names)}"
        h = C.c_void_p(0x5000 + len(names))
        names[h.value] = (tag, None)
        arr = np.asarray(arr, dtype=np.complex128) if kind == "numpy" else arr.numpy().astype(np.complex128)
        log.append((kind, tag, arr.shape, arr.tolist()))
        return DeviceTensor(ctx, h, arr.shape)

    def adopt(cls, ctx, h):
        tag, shape = names[h.value]
        log.append(("adopt", tag))
        return cls(ctx, C.c_void_p(h.value), shape)

    def to_numpy(self):
        log.append(("download", names[self.handle.value][0]))
        return np.zeros(self.shape, dtype=np.complex128)

    def free(self):
        if self.handle is not None:
            log.append(("free", names[self.handle.value][0]))
        self.handle = None

    class Stream:
        def __init__(self, name):
            self.name = name

        def wait_stream(self, other):
            log.append(("wait", self.name, other.name))

    monkeypatch.setattr(DeviceTensor, "from_numpy", classmethod(lambda cls, ctx, arr: make(ctx, arr, "numpy")))
    monkeypatch.setattr(DeviceTensor, "from_torch", classmethod(lambda cls, ctx, t: make(ctx, t, "torch")))
    monkeypatch.setattr(DeviceTensor, "adopt", classmethod(adopt))
    monkeypatch.setattr(DeviceTensor, "to_numpy", to_numpy)
    monkeypatch.setattr(DeviceTensor, "free", free)
    monkeypatch.setattr(tb, "torch_streams", lambda ctx: (Stream("torch"), Stream("ctx")))
    del log[:]
    yield plans, log, tn
    for p in plans.values():
        p = p.plan if hasattr(p, "plan") else p
        built_lib.tncb_plan_destroy(p.handle)
        p.handle = None


def arr(*shape, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(-3, 4, shape) + 1j * rng.integers(-3, 4, shape)


def cases(tn):
    """(name, plan kind, call) of every public method with host inputs, refusals included"""
    from tnc_b200.tensornetwork import Tensor
    tan = {0: arr(2, 3, seed=1), 2: arr(2, 2, seed=2)}
    rows = {0: arr(3, 2, 3, seed=3), 1: arr(3, 2, seed=4)}
    seed, seeds = arr(2, 2, seed=5), arr(3, 2, 2, seed=6)
    c = [("stage", "plain", lambda p: p.stage(tn)),
         ("run", "plain", lambda p: p.run().legs),
         ("execute", "plain", lambda p: p.execute(tn).legs),
         ("stage_slices", "plain", lambda p: p.stage_slices([tn, tn, tn])),
         ("run_slices", "plain", lambda p: p.run_slices(1, 2).legs),
         ("run_batch", "plain", lambda p: (p.stage_slices([tn, tn]), p.run_batch(1))[1][0]),
         ("run_batch count", "plain", lambda p: p.run_batch(0, 2)[0]),
         ("stage_instances", "plain", lambda p: (p.stage_instances(tn, {}, 4), p.n_staged)[1]),
         ("set_leaves", "vjp", lambda p: p.set_leaves({})),
         ("stage_instances bad leaf", "plain", lambda p: p.stage_instances(tn, {5: np.zeros(2)}, 2)),
         ("set_leaves host", "vjp", lambda p: p.set_leaves({1: np.zeros((3, 2))})),
         ("run vjp", "vjp", lambda p: p.run().legs),
         ("execute vjp", "vjp", lambda p: p.execute(tn).legs),
         ("vjp", "vjp", lambda p: p.vjp(seed)),
         ("vjp_block", "vjp", lambda p: p.vjp_block(seed).shape),
         ("stage_batch", "vjp", lambda p: (p.stage_batch([tn, tn, tn]), p.n_staged)[1]),
         ("vjp_batch", "vjp", lambda p: (p.stage_batch([tn, tn, tn]), p.vjp_batch(0, None, seeds, rows=True, sum=True))[1]),
         ("vjp_batch values", "vjp", lambda p: p.vjp_batch(1, 3, seeds, rows=False, sum=False, values=True)),
         ("vjp_batch sum", "vjp", lambda p: p.vjp_batch(0, 3, seeds, rows=False, sum=True, values=False)),
         ("vjp_batch_blocks", "vjp", lambda p: p.vjp_batch_blocks(0, 3, None, rows=True, sum=False, values=False)),
         ("jvp", "jvp", lambda p: p.jvp(tan)),
         ("jvp_block", "jvp", lambda p: p.jvp_block({}) and None),
         ("jvp_batch", "jvp", lambda p: (p.stage_batch([tn, tn, tn]), p.jvp_batch(0, None, rows))[1]),
         ("jvp_batch no values", "jvp", lambda p: p.jvp_batch(1, 3, rows, values=False)),
         ("jvp_batch no tangents", "jvp", lambda p: p.jvp_batch_blocks(0, 2, None)),
         ("hvp", "hvp", lambda p: p.hvp(tan, seed, arr(2, 2, seed=8))),
         ("hvp_blocks", "hvp", lambda p: p.hvp_blocks(tan, seed, None, outputs=(False, True, False, True))),
         ("hvp_blocks grads", "hvp", lambda p: p.hvp_blocks({}, None, seed, outputs=(True, False, True, False))),
         ("hvp_batch", "hvp", lambda p: p.hvp_batch(3, rows, seeds, seeds)),
         ("hvp_batch packed", "hvp", lambda p: p.hvp_batch(3, arr(3, 16, seed=9), seeds,
                                                           outputs=(False, False, True, True, False, True))),
         ("hvp_batch_blocks", "hvp", lambda p: p.hvp_batch_blocks(2, {1: arr(3, 2)}, None, None,
                                                                  outputs=(True, True, False, False, True, False))),
         ("hvp_batch bad tangents", "hvp", lambda p: p.hvp_batch_blocks(3, arr(3, 15))),
         ("hvp_batch bad seeds", "hvp", lambda p: p.hvp_batch_blocks(3, rows, arr(3, 2))),
         ("hvp_batch bad seed tangents", "hvp", lambda p: p.hvp_batch_blocks(3, rows, seeds, arr(2, 2, 2))),
         ("hvp_batch bad payload", "hvp", lambda p: p.hvp_batch_blocks(3, rows, seeds, payloads={3: np.zeros(2)})),
         ("hvp_batch host payload", "hvp", lambda p: p.hvp_batch_blocks(3, rows, seeds, payloads={0: np.zeros((2, 3))})),
         ("tangent bad leaf", "jvp", lambda p: p.jvp_block({3: np.zeros(2)})),
         ("tangent bad shape", "hvp", lambda p: p.hvp_blocks({0: np.zeros((3, 2))}, seed)),
         ("jvp_block no tangents", "jvp", lambda p: p.jvp_block(None)),
         ("hvp_blocks no tangents", "hvp", lambda p: p.hvp_blocks(None, seed)),
         ("hvp_batch no tangents", "hvp", lambda p: p.hvp_batch_blocks(2, None)),
         ("tangent rows bad shape", "jvp", lambda p: p.jvp_batch_blocks(0, 2, {0: np.zeros((3, 2, 3))})),
         ("sliced run", "sliced", lambda p: p.run().legs),
         ("sliced run world", "sliced", lambda p: p.run(1, 2).legs),
         ("sliced run no allreduce", "sliced", lambda p: p.run(0, 2, allreduce=False).legs),
         ("sliced set_leaves", "sliced", lambda p: p.set_leaves({})),
         ("sliced info", "sliced", lambda p: p.info()["pairs"]),
         ("sliced vjp stage", "sliced vjp", lambda p: p.stage(tn)),
         ("sliced vjp run", "sliced vjp", lambda p: p.run(0, 2).legs),
         ("sliced vjp_blocks", "sliced vjp", lambda p: [b.shape for b in p.vjp_blocks(seed, 1, 2)]),
         ("sliced vjp_blocks no allreduce", "sliced vjp", lambda p: [b.shape for b in p.vjp_blocks(None, 0, 2, False)]),
         ("sliced vjp", "sliced vjp", lambda p: p.vjp(seed, 1, 2)),
         ("sliced vjp again", "sliced vjp", lambda p: p.vjp(None)),
         ("sliced vjp set_leaves", "sliced vjp", lambda p: p.set_leaves({})),
         ("sliced jvp", "sliced jvp", lambda p: p.jvp(tan, 0, 3)),
         ("sliced jvp_block no tangents", "sliced jvp", lambda p: p.jvp_block(None)),
         ("sliced hvp_blocks no tangents", "sliced hvp", lambda p: p.hvp_blocks(None)),
         ("sliced jvp_block", "sliced jvp", lambda p: [b.shape for b in p.jvp_block({1: arr(3, 2)}, 1, 3, False)]),
         ("sliced hvp", "sliced hvp", lambda p: p.hvp(tan, seed, seed)),
         ("sliced hvp world", "sliced hvp", lambda p: p.hvp(tan, None, None, 1, 2)),
         ("sliced hvp_blocks", "sliced hvp", lambda p: p.hvp_blocks({}, seed, None, 0, 2, True, (True, False, False, True))),
         ("sliced hvp_blocks no allreduce", "sliced hvp", lambda p: p.hvp_blocks(tan, seed, None, 0, 2, False)),
         ("sliced grad_offsets", "sliced hvp", lambda p: p.grad_offsets())]
    return c


def summary(x):
    """a picklable, comparable summary of a return value"""
    if isinstance(x, np.ndarray):
        return ("array", x.shape)
    if isinstance(x, dict):
        return {k: summary(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [summary(v) for v in x]
    if type(x).__name__ == "DeviceTensor":
        return ("device", x.shape)
    if type(x).__name__ == "Tensor":
        return ("tensor", list(x.legs), list(x.bond_dims))
    return x


def run_case(plans, log, call, kind):
    """(the outcome, the log) of one call; the dummy handles renamed in order of appearance"""
    del log[:]
    try:
        got = ("ok", summary(call(plans[kind])))
    except Exception as e:                  # refusals: the type and the message
        got = ("raise", type(e).__name__, str(e))
    tags = {}

    def rename(x):
        if isinstance(x, str) and x[-1:].isdigit() and x.rstrip("0123456789") in ("up", "out"):
            kind = x.rstrip("0123456789")
            return tags.setdefault(x, f"{kind}{sum(t.startswith(kind) for t in tags.values())}")
        return x
    return got, [tuple(rename(x) for x in row) for row in log]


# recorded from the wrappers before they shared one call path; the one deliberate change: SlicedPlan.vjp reads the
# result's legs from the plan instead of running an empty slice range (tncb_plan_run_slices(n_slices, 1)) first
CALLS = {'stage': (('ok', None), [('tncb_plan_stage', 'plan', 'node')]),
 'run': (('ok', [3, 0]), [('tncb_plan_run', 'plan', 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'execute': (('ok', [3, 0]),
             [('tncb_plan_execute', 'plan', 'node', 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'stage_slices': (('ok', None), [('tncb_plan_stage_slices', 'plan', 3, ('nodes', 3))]),
 'run_slices': (('ok', [3, 0]),
                [('tncb_plan_run_slices', 'plan', 1, 2, 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'run_batch': (('ok', [3, 0]),
               [('tncb_plan_stage_slices', 'plan', 2, ('nodes', 2)),
                ('tncb_plan_run_batch', 'plan', 1, 1, 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'run_batch count': (('ok', [3, 0]),
                     [('tncb_plan_run_batch', 'plan', 0, 2, 'out', 'n_out', 'legs'), ('adopt', 'out0'),
                      ('free', 'out0')]),
 'stage_instances': (('ok', 4),
                     [('wait', 'ctx', 'torch'),
                      ('tncb_plan_stage_instances', 'plan', 'node', 4, 0, ('u64', [0]), ('ptrs', [None]), ('u64', [0])),
                      ('wait', 'torch', 'ctx')]),
 'set_leaves': (('ok', None),
                [('wait', 'ctx', 'torch'), ('tncb_plan_set_leaves', 'plan', 0, ('u64', [0]), ('ptrs', [None])),
                 ('wait', 'torch', 'ctx')]),
 'stage_instances bad leaf': (('raise', 'IndexError', 'leaf index 5 out of range (3 leaves)'), []),
 'set_leaves host': (('raise', 'ValueError', 'the payload of leaf 1 must be a torch CUDA tensor, got ndarray'), []),
 'run vjp': (('ok', [3, 0]), [('tncb_plan_run', 'plan', 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'execute vjp': (('ok', [3, 0]),
                 [('tncb_plan_execute', 'plan', 'node', 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'vjp': (('ok', {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}),
         [('numpy', 'up0', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]), ('tncb_plan_vjp', 'plan', 'up0', 'out'),
          ('free', 'up0'), ('adopt', 'out0'), ('download', 'out0'), ('free', 'out0')]),
 'vjp_block': (('ok', [16]),
               [('numpy', 'up0', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                ('tncb_plan_vjp', 'plan', 'up0', 'out'), ('free', 'up0'), ('adopt', 'out0'), ('free', 'out0')]),
 'stage_batch': (('ok', 3), [('tncb_plan_stage_batch', 'plan', 3, ('nodes', 3))]),
 'vjp_batch': (('ok',
                [[3, 0], ('array', (3, 2, 2)),
                 {0: ('array', (3, 2, 3)), 1: ('array', (3, 3, 2)), 2: ('array', (3, 2, 2))},
                 {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
               [('tncb_plan_stage_batch', 'plan', 3, ('nodes', 3)),
                ('numpy', 'up0', (3, 2, 2),
                 [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                  [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                ('tncb_plan_vjp_batch', 'plan', 0, 3, 'up0', 'out', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'),
                ('adopt', 'out1'), ('adopt', 'out2'), ('download', 'out0'), ('free', 'out0'), ('download', 'out1'),
                ('free', 'out1'), ('download', 'out2'), ('free', 'out2')]),
 'vjp_batch values': (('ok', [[3, 0], ('array', (3, 2, 2)), None, None]),
                      [('numpy', 'up0', (3, 2, 2),
                        [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                         [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                       ('tncb_plan_vjp_batch', 'plan', 1, 3, 'up0', 'out', None, None), ('free', 'up0'),
                       ('adopt', 'out0'), ('download', 'out0'), ('free', 'out0')]),
 'vjp_batch sum': (('ok', [[3, 0], None, None, {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
                   [('numpy', 'up0', (3, 2, 2),
                     [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                      [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                    ('tncb_plan_vjp_batch', 'plan', 0, 3, 'up0', None, None, 'out'), ('free', 'up0'), ('adopt', 'out0'),
                    ('download', 'out0'), ('free', 'out0')]),
 'vjp_batch_blocks': (('ok', [None, ('device', (3, 16)), None]),
                      [('tncb_plan_vjp_batch', 'plan', 0, 3, None, None, 'out', None), ('adopt', 'out0'),
                       ('free', 'out0')]),
 'jvp': (('ok', [('tensor', [3, 0], [2, 2]), ('array', (2, 2))]),
         [('numpy', 'up0', (16,),
           [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j), (-2+2j), (-3+0j), (-1-3j)]),
          ('tncb_plan_jvp', 'plan', 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'), ('adopt', 'out1'),
          ('download', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'jvp_block': (('ok', None),
               [('numpy', 'up0', (16,), [0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j]),
                ('tncb_plan_jvp', 'plan', 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'), ('adopt', 'out1'),
                ('free', 'out1'), ('free', 'out0')]),
 'jvp_batch': (('ok', [[3, 0], ('array', (3, 2, 2)), ('array', (3, 2, 2))]),
               [('tncb_plan_stage_batch', 'plan', 3, ('nodes', 3)),
                ('numpy', 'up0', (3, 16),
                 [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j), 0j,
                   0j, 0j, 0j],
                  [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j), 0j, 0j,
                   0j, 0j],
                  [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j), 0j, 0j, 0j,
                   0j]]),
                ('tncb_plan_jvp_batch', 'plan', 0, 3, 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'),
                ('adopt', 'out1'), ('download', 'out0'), ('free', 'out0'), ('download', 'out1'), ('free', 'out1')]),
 'jvp_batch no values': (('ok', [[3, 0], None, ('array', (3, 2, 2))]),
                         [('numpy', 'up0', (3, 16),
                           [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                             (3-1j), 0j, 0j, 0j, 0j],
                            [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j),
                             0j, 0j, 0j, 0j],
                            [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j),
                             0j, 0j, 0j, 0j]]),
                          ('tncb_plan_jvp_batch', 'plan', 1, 3, 'up0', None, 'out'), ('free', 'up0'), ('adopt', 'out0'),
                          ('download', 'out0'), ('free', 'out0')]),
 'jvp_batch no tangents': (('ok', [('device', (2, 2, 2)), ('device', (2, 2, 2))]),
                           [('numpy', 'up0', (2, 16),
                             [[0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j],
                              [0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j]]),
                            ('tncb_plan_jvp_batch', 'plan', 0, 2, 'up0', 'out', 'out'), ('free', 'up0'),
                            ('adopt', 'out0'), ('adopt', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'hvp': (('ok',
          [('array', (2, 2)), ('array', (2, 2)), {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))},
           {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
         [('numpy', 'up0', (16,),
           [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j), (-2+2j), (-3+0j), (-1-3j)]),
          ('numpy', 'up1', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
          ('numpy', 'up2', (2, 2), [[(2-2j), (-1-1j)], [(-2+1j), (3+2j)]]),
          ('tncb_plan_hvp', 'plan', 'up0', 'up1', 'up2', 'out', 'out', 'out', 'out'), ('free', 'up0'), ('free', 'up1'),
          ('free', 'up2'), ('adopt', 'out0'), ('adopt', 'out1'), ('adopt', 'out2'), ('adopt', 'out3'),
          ('download', 'out0'), ('free', 'out0'), ('download', 'out1'), ('free', 'out1'), ('download', 'out2'),
          ('free', 'out2'), ('download', 'out3'), ('free', 'out3')]),
 'hvp_blocks': (('ok', [None, ('device', (2, 2)), None, ('device', (16,))]),
                [('numpy', 'up0', (16,),
                  [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j), (-2+2j), (-3+0j),
                   (-1-3j)]),
                 ('numpy', 'up1', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                 ('tncb_plan_hvp', 'plan', 'up0', 'up1', None, None, 'out', None, 'out'), ('free', 'up0'),
                 ('free', 'up1'), ('adopt', 'out0'), ('adopt', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'hvp_blocks grads': (('ok', [('device', (2, 2)), None, ('device', (16,)), None]),
                      [('numpy', 'up0', (16,), [0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j]),
                       ('numpy', 'up1', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                       ('tncb_plan_hvp', 'plan', 'up0', None, 'up1', 'out', None, 'out', None), ('free', 'up0'),
                       ('free', 'up1'), ('adopt', 'out0'), ('adopt', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'hvp_batch': (('ok',
                [[3, 0], ('array', (3, 2, 2)), ('array', (3, 2, 2)),
                 {0: ('array', (3, 2, 3)), 1: ('array', (3, 3, 2)), 2: ('array', (3, 2, 2))},
                 {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))},
                 {0: ('array', (3, 2, 3)), 1: ('array', (3, 3, 2)), 2: ('array', (3, 2, 2))},
                 {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
               [('numpy', 'up0', (3, 16),
                 [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j), 0j,
                   0j, 0j, 0j],
                  [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j), 0j, 0j,
                   0j, 0j],
                  [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j), 0j, 0j, 0j,
                   0j]]),
                ('numpy', 'up1', (3, 2, 2),
                 [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                  [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                ('numpy', 'up2', (3, 2, 2),
                 [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                  [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                ('tncb_plan_hvp_batch', 'plan', 3, 0, ('u64', [0]), ('ptrs', [None]), ('u64', [0]), 'up0', 'up1', 'up2',
                 'out', 'out', 'out', 'out', 'out', 'out'),
                ('free', 'up0'), ('free', 'up1'), ('free', 'up2'), ('adopt', 'out0'), ('adopt', 'out1'),
                ('adopt', 'out2'), ('adopt', 'out3'), ('adopt', 'out4'), ('adopt', 'out5'), ('download', 'out0'),
                ('free', 'out0'), ('download', 'out1'), ('free', 'out1'), ('download', 'out2'), ('free', 'out2'),
                ('download', 'out3'), ('free', 'out3'), ('download', 'out4'), ('free', 'out4'), ('download', 'out5'),
                ('free', 'out5')]),
 'hvp_batch packed': (('ok',
                       [[3, 0], None, None, {0: ('array', (3, 2, 3)), 1: ('array', (3, 3, 2)), 2: ('array', (3, 2, 2))},
                        {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}, None,
                        {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
                      [('numpy', 'up0', (3, 16),
                        [[(-1-3j), (3+3j), (3+3j), (-1+3j), (-3+3j), (1+1j), (1+1j), (2+0j), (1-3j), (2+3j), (3+3j),
                          (3-3j), (3+1j), (3-1j), (2+2j), (3+1j)],
                         [(-3+1j), (-3+0j), (2-3j), 2j, (2+3j), -2j, (3+0j), (-3-3j), (1+0j), (-3-3j), (-2-1j), (2+3j),
                          (-1-3j), (3-3j), (-1+1j), (2-2j)],
                         [(3-3j), (-1-1j), (3-2j), (1+1j), (3+0j), (-1+2j), 1j, (2-3j), (3-3j), (-2+3j), 2j, (2+2j),
                          (2+2j), (3-1j), (-2+0j), (3-2j)]]),
                       ('numpy', 'up1', (3, 2, 2),
                        [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                         [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                       ('tncb_plan_hvp_batch', 'plan', 3, 0, ('u64', [0]), ('ptrs', [None]), ('u64', [0]), 'up0', 'up1',
                        None, None, None, 'out', 'out', None, 'out'),
                       ('free', 'up0'), ('free', 'up1'), ('adopt', 'out0'), ('adopt', 'out1'), ('adopt', 'out2'),
                       ('download', 'out0'), ('free', 'out0'), ('download', 'out1'), ('free', 'out1'),
                       ('download', 'out2'), ('free', 'out2')]),
 'hvp_batch_blocks': (('ok', [('device', (2, 2, 2)), ('device', (2, 2, 2)), None, None, ('device', (2, 16)), None]),
                      [('numpy', 'up0', (2, 16),
                        [[0j, 0j, 0j, 0j, 0j, 0j, (2-3j), (1-3j), -2j, (-2+2j), (-1+1j), (-3+3j), 0j, 0j, 0j, 0j],
                         [0j, 0j, 0j, 0j, 0j, 0j, (2-3j), (1-3j), -2j, (-2+2j), (-1+1j), (-3+3j), 0j, 0j, 0j, 0j]]),
                       ('tncb_plan_hvp_batch', 'plan', 2, 0, ('u64', [0]), ('ptrs', [None]), ('u64', [0]), 'up0', None,
                        None, 'out', 'out', None, None, 'out', None),
                       ('free', 'up0'), ('adopt', 'out0'), ('adopt', 'out1'), ('adopt', 'out2'), ('free', 'out2'),
                       ('free', 'out1'), ('free', 'out0')]),
 'hvp_batch bad tangents': (('raise', 'ValueError', 'the tangents have shape (3, 15), expected (3, 16)'), []),
 'hvp_batch bad seeds': (('raise', 'ValueError', 'the seeds have shape (3, 2), expected (3, 2, 2)'),
                         [('numpy', 'up0', (3, 16),
                           [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                             (3-1j), 0j, 0j, 0j, 0j],
                            [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j),
                             0j, 0j, 0j, 0j],
                            [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j),
                             0j, 0j, 0j, 0j]]),
                          ('free', 'up0')]),
 'hvp_batch bad seed tangents': (('raise', 'ValueError', 'the seed tangents have shape (2, 2, 2), expected (3, 2, 2)'),
                                 [('numpy', 'up0', (3, 16),
                                   [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j,
                                     (3-2j), (3-1j), 0j, 0j, 0j, 0j],
                                    [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                                     (3-1j), 0j, 0j, 0j, 0j],
                                    [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                                     (3-1j), 0j, 0j, 0j, 0j]]),
                                  ('numpy', 'up1', (3, 2, 2),
                                   [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                                    [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                                  ('free', 'up0'), ('free', 'up1')]),
 'hvp_batch bad payload': (('raise', 'IndexError', 'leaf index 3 out of range (3 leaves)'),
                           [('numpy', 'up0', (3, 16),
                             [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                               (3-1j), 0j, 0j, 0j, 0j],
                              [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                               (3-1j), 0j, 0j, 0j, 0j],
                              [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j), (3-1j),
                               0j, 0j, 0j, 0j]]),
                            ('numpy', 'up1', (3, 2, 2),
                             [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                              [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                            ('free', 'up0'), ('free', 'up1')]),
 'hvp_batch host payload': (('raise', 'ValueError', 'the payload of leaf 0 must be a torch CUDA tensor, got ndarray'),
                            [('numpy', 'up0', (3, 16),
                              [[(2-3j), (-3-3j), (-2+0j), (-2-1j), (-2+3j), (2+0j), (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                                (3-1j), 0j, 0j, 0j, 0j],
                               [(3-1j), (1+0j), (-3+1j), (-3+1j), (-1-2j), 2j, (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                                (3-1j), 0j, 0j, 0j, 0j],
                               [(1+2j), 3j, (-2+2j), (-2-2j), (1-1j), (2+1j), (2+3j), (3-3j), (3+0j), 1j, (3-2j),
                                (3-1j), 0j, 0j, 0j, 0j]]),
                             ('numpy', 'up1', (3, 2, 2),
                              [[[-1j, 1j], [2j, (-1-1j)]], [[(3+1j), (-1+1j)], [(1+0j), (-1-3j)]],
                               [[1j, (3-3j)], [(-2+3j), (1+2j)]]]),
                             ('free', 'up0'), ('free', 'up1')]),
 'tangent bad leaf': (('raise', 'IndexError', 'leaf index 3 out of range (3 leaves)'), []),
 'tangent bad shape': (('raise', 'ValueError', 'the tangent of leaf 0 has shape (3, 2), expected (2, 3)'), []),
 'jvp_block no tangents': (('raise', 'AttributeError', "'NoneType' object has no attribute 'values'"), []),
 'hvp_blocks no tangents': (('raise', 'AttributeError', "'NoneType' object has no attribute 'values'"), []),
 'hvp_batch no tangents': (('ok',
                            [('device', (2, 2, 2)), ('device', (2, 2, 2)), ('device', (2, 16)), ('device', (16,)),
                             ('device', (2, 16)), ('device', (16,))]),
                           [('tncb_plan_hvp_batch', 'plan', 2, 0, ('u64', [0]), ('ptrs', [None]), ('u64', [0]), None,
                             None, None, 'out', 'out', 'out', 'out', 'out', 'out'),
                            ('adopt', 'out0'), ('adopt', 'out1'), ('adopt', 'out2'), ('adopt', 'out3'),
                            ('adopt', 'out4'), ('adopt', 'out5'), ('free', 'out5'), ('free', 'out4'), ('free', 'out3'),
                            ('free', 'out2'), ('free', 'out1'), ('free', 'out0')]),
 'tangent rows bad shape': (('raise', 'ValueError',
                             'the tangent of leaf 0 has shape (3, 2, 3), expected (2, 2, 3) or (2, 3)'),
                            []),
 'sliced run': (('ok', [3, 0]),
                [('tncb_plan_run_slices', 'plan', 0, 1, 'out', 'n_out', 'legs'), ('adopt', 'out0'), ('free', 'out0')]),
 'sliced run world': (('ok', [3, 0]),
                      [('tncb_plan_run_slices', 'plan', 1, 2, 'out', 'n_out', 'legs'), ('adopt', 'out0'),
                       ('tncb_comm_allreduce_sum', 'out0'), ('free', 'out0')]),
 'sliced run no allreduce': (('ok', [3, 0]),
                             [('tncb_plan_run_slices', 'plan', 0, 2, 'out', 'n_out', 'legs'), ('adopt', 'out0'),
                              ('free', 'out0')]),
 'sliced set_leaves': (('raise', 'TypeError',
                        'set_leaves needs a sliced gradient plan (SlicedPlan.for_gradients); this plan stages every '
                        'slice on the host'),
                       []),
 'sliced info': (('ok', 2), []),
 'sliced vjp stage': (('ok', None), [('tncb_plan_stage', 'plan', 'node')]),
 'sliced vjp run': (('ok', [3, 0]),
                    [('tncb_plan_run_slices', 'plan', 0, 2, 'out', 'n_out', 'legs'), ('adopt', 'out0'),
                     ('tncb_comm_allreduce_sum', 'out0'), ('free', 'out0')]),
 'sliced vjp_blocks': (('ok', [[2, 2], [16]]),
                       [('numpy', 'up0', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                        ('tncb_plan_vjp_sliced', 'plan', 1, 2, 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'),
                        ('adopt', 'out1'), ('tncb_comm_allreduce_sum', 'out0'), ('tncb_comm_allreduce_sum', 'out1'),
                        ('free', 'out0'), ('free', 'out1')]),
 'sliced vjp_blocks no allreduce': (('ok', [[2, 2], [16]]),
                                    [('tncb_plan_vjp_sliced', 'plan', 0, 2, None, 'out', 'out'), ('adopt', 'out0'),
                                     ('adopt', 'out1'), ('free', 'out0'), ('free', 'out1')]),
 'sliced vjp': (('ok',
                 [('tensor', [3, 0], [2, 2]), {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
                [('numpy', 'up0', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                 ('tncb_plan_vjp_sliced', 'plan', 1, 2, 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'),
                 ('adopt', 'out1'), ('tncb_comm_allreduce_sum', 'out0'), ('tncb_comm_allreduce_sum', 'out1'),
                 ('download', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'sliced vjp again': (('ok',
                       [('tensor', [3, 0], [2, 2]),
                        {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
                      [('tncb_plan_vjp_sliced', 'plan', 0, 1, None, 'out', 'out'), ('adopt', 'out0'), ('adopt', 'out1'),
                       ('download', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'sliced vjp set_leaves': (('ok', None),
                           [('wait', 'ctx', 'torch'),
                            ('tncb_plan_set_leaves', 'plan', 0, ('u64', [0]), ('ptrs', [None])),
                            ('wait', 'torch', 'ctx')]),
 'sliced jvp': (('ok', [('tensor', [3, 0], [2, 2]), ('array', (2, 2))]),
                [('numpy', 'up0', (16,),
                  [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j), (-2+2j), (-3+0j),
                   (-1-3j)]),
                 ('tncb_plan_jvp_sliced', 'plan', 0, 3, 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'),
                 ('adopt', 'out1'), ('tncb_comm_allreduce_sum', 'out0'), ('tncb_comm_allreduce_sum', 'out1'),
                 ('download', 'out1'), ('free', 'out1'), ('free', 'out0')]),
 'sliced jvp_block no tangents': (('raise', 'AttributeError', "'NoneType' object has no attribute 'values'"), []),
 'sliced hvp_blocks no tangents': (('raise', 'AttributeError', "'NoneType' object has no attribute 'values'"), []),
 'sliced jvp_block': (('ok', [[2, 2], [2, 2]]),
                      [('numpy', 'up0', (16,),
                        [0j, 0j, 0j, 0j, 0j, 0j, (2-3j), (1-3j), -2j, (-2+2j), (-1+1j), (-3+3j), 0j, 0j, 0j, 0j]),
                       ('tncb_plan_jvp_sliced', 'plan', 1, 3, 'up0', 'out', 'out'), ('free', 'up0'), ('adopt', 'out0'),
                       ('adopt', 'out1'), ('free', 'out0'), ('free', 'out1')]),
 'sliced hvp': (('ok',
                 [('array', (2, 2)), ('array', (2, 2)),
                  {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))},
                  {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
                [('numpy', 'up0', (16,),
                  [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j), (-2+2j), (-3+0j),
                   (-1-3j)]),
                 ('numpy', 'up1', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                 ('numpy', 'up2', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                 ('tncb_plan_hvp_sliced', 'plan', 0, 1, 'up0', 'up1', 'up2', 'out', 'out', 'out', 'out'),
                 ('free', 'up0'), ('free', 'up1'), ('free', 'up2'), ('adopt', 'out0'), ('adopt', 'out1'),
                 ('adopt', 'out2'), ('adopt', 'out3'), ('download', 'out0'), ('free', 'out0'), ('download', 'out1'),
                 ('free', 'out1'), ('download', 'out2'), ('free', 'out2'), ('download', 'out3'), ('free', 'out3')]),
 'sliced hvp world': (('ok',
                       [('array', (2, 2)), ('array', (2, 2)),
                        {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))},
                        {0: ('array', (2, 3)), 1: ('array', (3, 2)), 2: ('array', (2, 2))}]),
                      [('numpy', 'up0', (16,),
                        [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j), (-2+2j), (-3+0j),
                         (-1-3j)]),
                       ('tncb_plan_hvp_sliced', 'plan', 1, 2, 'up0', None, None, 'out', 'out', 'out', 'out'),
                       ('free', 'up0'), ('adopt', 'out0'), ('adopt', 'out1'), ('adopt', 'out2'), ('adopt', 'out3'),
                       ('tncb_comm_allreduce_sum', 'out0'), ('tncb_comm_allreduce_sum', 'out1'),
                       ('tncb_comm_allreduce_sum', 'out2'), ('tncb_comm_allreduce_sum', 'out3'), ('download', 'out0'),
                       ('free', 'out0'), ('download', 'out1'), ('free', 'out1'), ('download', 'out2'), ('free', 'out2'),
                       ('download', 'out3'), ('free', 'out3')]),
 'sliced hvp_blocks': (('ok', [('device', (2, 2)), None, None, ('device', (16,))]),
                       [('numpy', 'up0', (16,), [0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j, 0j]),
                        ('numpy', 'up1', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                        ('tncb_plan_hvp_sliced', 'plan', 0, 2, 'up0', 'up1', None, 'out', None, None, 'out'),
                        ('free', 'up0'), ('free', 'up1'), ('adopt', 'out0'), ('adopt', 'out1'),
                        ('tncb_comm_allreduce_sum', 'out0'), ('tncb_comm_allreduce_sum', 'out1'), ('free', 'out1'),
                        ('free', 'out0')]),
 'sliced hvp_blocks no allreduce': (('ok',
                                     [('device', (2, 2)), ('device', (2, 2)), ('device', (16,)), ('device', (16,))]),
                                    [('numpy', 'up0', (16,),
                                      [2j, 3j, (2-2j), (3-1j), (-3+3j), (-2-1j), 0j, 0j, 0j, 0j, 0j, 0j, (2-1j),
                                       (-2+2j), (-3+0j), (-1-3j)]),
                                     ('numpy', 'up1', (2, 2), [[(1+0j), (2+0j)], [(-3+1j), (2-1j)]]),
                                     ('tncb_plan_hvp_sliced', 'plan', 0, 2, 'up0', 'up1', None, 'out', 'out', 'out',
                                      'out'),
                                     ('free', 'up0'), ('free', 'up1'), ('adopt', 'out0'), ('adopt', 'out1'),
                                     ('adopt', 'out2'), ('adopt', 'out3'), ('free', 'out3'), ('free', 'out2'),
                                     ('free', 'out1'), ('free', 'out0')]),
 'sliced grad_offsets': (('ok', [0, 6, 12]), [])}


def test_calls(rec):
    plans, log, tn = rec
    got = {name: run_case(plans, log, call, kind) for name, kind, call in cases(tn)}
    assert list(got) == list(CALLS)
    for name, want in CALLS.items():
        assert got[name] == want, name


def test_torch_seeds(rec):
    """seeds of every vjp are converted as the hvp seeds are: a torch tensor goes through DeviceTensor.from_torch, which
    takes only CUDA tensors (here the CPU one is recorded as if it were one)"""
    import torch
    plans, log, tn = rec
    seed, seeds = torch.ones((2, 2), dtype=torch.complex128), torch.ones((3, 2, 2), dtype=torch.complex128)
    plans["vjp"].stage_batch([tn, tn, tn])
    for kind, call, want in (("vjp", lambda p: p.vjp_block(seed), "tncb_plan_vjp"),
                             ("vjp", lambda p: p.vjp(seed), "tncb_plan_vjp"),
                             ("vjp", lambda p: p.vjp_batch_blocks(0, 3, seeds), "tncb_plan_vjp_batch"),
                             ("vjp", lambda p: p.vjp_batch(0, None, seeds), "tncb_plan_vjp_batch"),
                             ("sliced vjp", lambda p: p.vjp_blocks(seed), "tncb_plan_vjp_sliced"),
                             ("sliced vjp", lambda p: p.vjp(seed), "tncb_plan_vjp_sliced")):
        got, entries = run_case(plans, log, call, kind)
        assert got[0] == "ok", got
        assert entries[0][:3] == ("torch", "up0", tuple(seed.shape) if "batch" not in want else (3, 2, 2))
        assert entries[1][0] == want and "up0" in entries[1] and ("free", "up0") in entries


def test_packed_tangents(rec):
    """every jvp and hvp takes the tangents packed at grad_offsets(), uploaded as they are; a DeviceTensor passes through"""
    from tnc_b200 import DeviceTensor
    plans, log, tn = rec
    block, rows = arr(16, seed=11), arr(3, 16, seed=12)
    dev = DeviceTensor(None, C.c_void_p(0x9000), (16,))
    plans["jvp"].stage_batch([tn, tn, tn])
    for kind, call, x in (("jvp", lambda p: p.jvp_block(block), block), ("jvp", lambda p: p.jvp(block), block),
                          ("jvp", lambda p: p.jvp_batch_blocks(0, 3, rows), rows), ("jvp", lambda p: p.jvp_batch(0, 3, rows), rows),
                          ("hvp", lambda p: p.hvp_blocks(block), block), ("hvp", lambda p: p.hvp(block), block),
                          ("sliced jvp", lambda p: p.jvp_block(block), block), ("sliced jvp", lambda p: p.jvp(block), block),
                          ("sliced hvp", lambda p: p.hvp_blocks(block), block), ("sliced hvp", lambda p: p.hvp(block), block)):
        got, entries = run_case(plans, log, call, kind)
        assert got[0] == "ok", got
        assert entries[0] == ("numpy", "up0", x.shape, x.tolist())
        assert "up0" in entries[1] and ("free", "up0") in entries
    got, entries = run_case(plans, log, lambda p: p.jvp_block(dev), "jvp")
    assert got[0] == "ok" and entries[0] == ("tncb_plan_jvp", "plan", "handle", "out", "out")
    for kind, call, what in (("jvp", lambda p: p.jvp_block(arr(15)), "(15,), expected (16,)"),
                             ("jvp", lambda p: p.jvp_batch_blocks(0, 3, arr(16)), "(16,), expected (3, 16)"),
                             ("sliced hvp", lambda p: p.hvp_blocks(arr(3, 16)), "(3, 16), expected (16,)")):
        assert run_case(plans, log, call, kind) == (("raise", "ValueError", f"the tangents have shape {what}"), []), kind


def test_host_seed_shapes(rec):
    """a host seed or seed tangent of the wrong shape is refused before it is uploaded, in every call"""
    plans, log, tn = rec
    plans["vjp"].stage_batch([tn, tn, tn])
    tan = {0: arr(2, 3)}
    for kind, call, msg in (
            ("vjp", lambda p: p.vjp_block(arr(4)), "the seed has shape (4,), the result (2, 2)"),
            ("vjp", lambda p: p.vjp(arr(2, 2, 1)), "the seed has shape (2, 2, 1), the result (2, 2)"),
            ("vjp", lambda p: p.vjp_batch_blocks(0, 3, arr(2, 2, 2)), "the seeds have shape (2, 2, 2), expected (3, 2, 2)"),
            ("vjp", lambda p: p.vjp_batch(0, None, arr(3, 4)), "the seeds have shape (3, 4), expected (3, 2, 2)"),
            ("hvp", lambda p: p.hvp_blocks(tan, arr(2)), "the seed has shape (2,), the result (2, 2)"),
            ("hvp", lambda p: p.hvp(tan, arr(2, 2), arr(4)), "the seed tangent has shape (4,), the result (2, 2)"),
            ("sliced vjp", lambda p: p.vjp_blocks(arr(2, 3)), "the seed has shape (2, 3), the result (2, 2)"),
            ("sliced vjp", lambda p: p.vjp(arr(1)), "the seed has shape (1,), the result (2, 2)"),
            ("sliced hvp", lambda p: p.hvp_blocks(tan, None, arr(2)), "the seed tangent has shape (2,), the result (2, 2)")):
        got, entries = run_case(plans, log, call, kind)
        assert got == ("raise", "ValueError", msg), (kind, got)
        refused = msg.split(" has shape ")[-1].split(" have shape ")[-1].split("),")[0] + ")"
        uploads = [e for e in entries if e[0] == "numpy"]
        assert all(str(e[2]) != refused and ("free", e[1]) in entries for e in uploads), entries
        assert all(not e[0].startswith("tncb_") for e in entries), entries
