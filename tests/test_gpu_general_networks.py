"""Every plan kind on general tensor networks, against one torch reference.

The other derivative and batch tests run random-circuit networks: every leg has dimension 2 (a few many-group cases
have one dimension-3 leg), every sliced leg has dimension 2 and no test builds a nested network for a gradient,
tangent, Hessian-vector, batched or sliced-gradient plan.  When all extents are equal, code that reads the extent of the
wrong leg, swaps two legs of equal extent or takes a slice digit as a bit still gives the right numbers.  This file runs
a seeded corpus of general networks instead:

  1. The corpus (no GPU).  24 networks with bond dimensions from {1, 2, 3, 5, 7} and a few legs of 64, leaves of rank
     0 to 8 and two of rank 10 and 12, scalar results and results of rank 1 to 6, two disconnected components
     joined by an outer product, flat greedy and random-order paths, and nested paths (built by hand, with
     partition_tensor_network, two levels deep, with single-leaf composites).  Payloads are random complex with each
     leaf scaled by 2^e, e in [-8, 8].  A host test pins what the corpus reaches: forward pairs and restated backward
     pairs classified by tncb_pair_kernel_class, their counts and flops against tncb_plan_info of host-only plans, K0,
     K1 and K2 with a K2 pair whose big side is not a power of two, and leaf adjoints that need more than 8 fused groups
     (K3).  K0 split-K, the int8 engine and K3 are chosen at launch; the GPU tests assert them with the engine counters.
  2. The reference (no GPU).  A complex128 torch TTGT replay that follows the path, nested or flat; G from
     torch.autograd.grad (conjugated), Ṙ from torch.func.jvp, Ġ from jvp of vjp; sliced references cut each slice with
     numpy indexing (slice q = the row-major digit vector over the sliced legs, last leg fastest), replay exactly the
     requested slices and embed the results back into full leaf shapes.  It is checked against a path-independent
     np.einsum of the whole network, and the sliced reference folded over every slice against the unsliced one.
  3. Every plan kind (GPU): forward (contract_tensor_network twice, stage + run, execute, the pair-by-pair executor),
     run_batch / run_slices, gradients (every leaf, a subset, one leaf deep inside a nested composite), vjp_batch rows and
     sum, jvp and jvp_batch over stride-0 directions, hvp with a seed tangent, sliced gradients on 1 to 3 mixed-radix
     legs (full range, single slices with non-zero digits, a (rank, world) sub-range), the forward SlicedPlan on flat
     networks, and device staging against host staging.  Errors are measured per output tensor and per leaf, in units of
     that tensor's largest reference entry: TAU = 1e-12 on FP64 routes; where the int8 engine ran, its tcgen05_bound
     at the pairs' contraction lengths plus the FP64 allowance.
  4. The comparator (no GPU) rejects, on the corpus references, a (3, 5) leaf gradient read with the extents of (5, 3),
     slice digits taken as bits, and a 1e-9 relative change of one entry of the smallest leaf's gradient; the first two
     pass when every extent is 2.
  5. The C++ mirror (tnc::NetworkPlan in include/tnc.hpp): its ForGradients / ForTangents / ForHvp methods on a nested,
     mixed-dimension network (tests/cpp/test_host_api.cpp --deriv) give bit for bit the blocks of the Python plans."""
import ctypes as C
import functools
import itertools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU = 1e-12
POOL = (1, 2, 3, 5, 7)
COUNTERS = ("k0", "k0_splitk", "k1_dmma", "k1_dmma_splitk", "k1_tcgen05", "k2", "permute")


# ================================================================================================================
# 1. the corpus
# ================================================================================================================
class Net:
    """a network of the corpus: tn (Tensor tree), path, and what the tests do with it.
    sliced: leg lists to slice; int8: run under set_tcgen05_threshold(1, 128); routes: engine counters its forward and
    backward passes must reach; deep: one leaf index deep inside a nested composite"""

    def __init__(self, name, tn, path, sliced=(), int8=False, routes=(), deep=None):
        from tnc_b200.tensornetwork import leaves
        self.name, self.tn, self.path = name, tn, path
        self.sliced, self.int8, self.routes = [list(s) for s in sliced], int8, set(routes)
        self.leaves = leaves(tn)
        self.flat = not path.nested
        self.deep = deep if deep is not None else len(self.leaves) - 1
        self.xs = [np.asarray(l.tensordata.matrix, dtype=np.complex128) for l in self.leaves]
        self.dim = {l: d for t in self.leaves for l, d in zip(t.legs, t.bond_dims)}


def crandn(rng, shape):
    return np.asarray(rng.standard_normal(shape) + 1j * rng.standard_normal(shape), dtype=np.complex128)


def matrix_leaf(legs, dims, x):
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    t = Tensor(list(legs), list(dims))
    t.set_tensor_data(TensorData.Matrix(np.asarray(x, dtype=np.complex128).reshape([int(d) for d in dims])))
    return t


def make_leaves(legs_list, dim, rng):
    """Matrix leaves with random complex payloads, each scaled by 2^e, e in [-8, 8]"""
    out = []
    for legs in legs_list:
        shape = [dim[l] for l in legs]
        out.append(matrix_leaf(legs, shape, crandn(rng, shape) * 2.0 ** int(rng.integers(-8, 9))))
    return out


def ext_legs(t):
    """{leg: dim} of the legs a (sub)network leaves open: every leg joins at most two tensors"""
    if not t.tensors:
        return dict(zip(t.legs, t.bond_dims))
    out = {}
    for c in t.tensors:
        for l, d in ext_legs(c).items():
            if l in out:
                del out[l]
            else:
                out[l] = d
    return out


def order(ops, rng, kind):
    """replace-left pairs over the operands ops ({leg: dim} each): greedy by output size, or random among the pairs that
    share a leg (any pair once none does)"""
    live = dict(enumerate(ops))
    pairs = []
    while len(live) > 1:
        keys = sorted(live)
        cand = list(itertools.combinations(keys, 2))
        joined = [(i, j) for i, j in cand if set(live[i]) & set(live[j])]
        if kind == "random":
            pool = joined or cand
            i, j = pool[int(rng.integers(len(pool)))]
        else:
            def cost(p):
                a, b = live[p[0]], live[p[1]]
                out = [d for l, d in a.items() if l not in b] + [d for l, d in b.items() if l not in a]
                return (0 if p in joined else 1, float(np.prod(out)), p)
            i, j = min(cand, key=cost)
        a, b = live[i], live[j]
        live[i] = {**{l: d for l, d in b.items() if l not in a}, **{l: d for l, d in a.items() if l not in b}}
        del live[j]
        pairs.append((i, j))
    return pairs


def tree_path(t, rng, kind="greedy"):
    """a replace-left path for the tree t: every composite child gets its own nested path (single-leaf composites an
    empty one), the children are ordered by `order`"""
    from tnc_b200.contractionpath import ContractionPath
    nested = {i: tree_path(c, rng, kind) for i, c in enumerate(t.tensors) if c.tensors}
    return ContractionPath(nested, order([ext_legs(c) for c in t.tensors], rng, kind))


def build_tree(leaves, groups):
    """groups: an int (that leaf) or a list of groups (a composite of them)"""
    from tnc_b200.tensornetwork import Tensor
    if isinstance(groups, int):
        return leaves[groups]
    return Tensor.new_composite([build_tree(leaves, g) for g in groups])


def random_structure(rng, n, extra, n_open, pool=POOL, weights=None, components=1, n_rank0=0, max_rank=8):
    """leg lists of n leaves: a spanning forest of `components` trees, `extra` more bonds inside components, n_open open
    legs, n_rank0 leaves without legs; every leg joins at most two leaves"""
    dim, legs = {}, [[] for _ in range(n)]
    nl = itertools.count()
    comp = np.array_split(np.arange(n), components)

    def add(ls, d):
        l = next(nl)
        dim[l] = int(d)
        for i in ls:
            legs[i].append(l)

    pick = lambda: rng.choice(pool, p=weights)
    for block in comp:
        for k in range(1, len(block)):
            prev = [int(j) for j in block[:k] if len(legs[j]) < max_rank]
            add((int(block[k]), prev[int(rng.integers(len(prev)))]), pick())
    for _ in range(extra):
        block = comp[int(rng.integers(components))]
        if len(block) < 2:
            continue
        i, j = (int(v) for v in rng.choice(block, 2, replace=False))
        if len(legs[i]) < max_rank and len(legs[j]) < max_rank:
            add((i, j), pick())
    for _ in range(n_open):
        i = int(rng.integers(n))
        if len(legs[i]) < max_rank:
            add((i,), pick())
    for ls in legs:
        rng.shuffle(ls)
    return legs + [[] for _ in range(n_rank0)], dim


def bonds_of(net, want):
    """bond legs (joining two leaves) with the extents `want`, in that order, distinct; None if the network lacks one"""
    count = {}
    for t in net.leaves:
        for l in t.legs:
            count[l] = count.get(l, 0) + 1
    out = []
    for d in want:
        hit = [l for l in sorted(count) if count[l] == 2 and net.dim[l] == d and l not in out]
        if not hit:
            return None
        out.append(hit[0])
    return out


def random_net(name, seed, n, extra, n_open, kind="greedy", groups=None, partition=None, components=1, n_rank0=0,
               weights=None, slice_extents=((3,), (5, 2), (3, 2, 5))):
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.partitioning import partition_tensor_network
    rng = np.random.default_rng(seed)
    legs, dim = random_structure(rng, n, extra, n_open, weights=weights, components=components, n_rank0=n_rank0)
    lv = make_leaves(legs, dim, rng)
    deep = None
    if partition is not None:
        tn = partition_tensor_network(Tensor.new_composite(lv), partition)
    elif groups is not None:
        tn = build_tree(lv, groups)
    else:
        tn = Tensor.new_composite(lv)
    path = tree_path(tn, rng, kind)
    if groups is not None or partition is not None:
        deep = deepest_leaf(tn)
    net = Net(name, tn, path, deep=deep, routes={"k0"})
    net.sliced = [s for s in (bonds_of(net, e) for e in slice_extents) if s]
    return net


def deepest_leaf(tn):
    """index (depth-first) of the first leaf at the greatest nesting depth"""
    best, idx = (-1, 0), [0]

    def walk(t, depth):
        nonlocal best
        if not t.tensors:
            if depth > best[0]:
                best = (depth, idx[0])
            idx[0] += 1
            return
        for c in t.tensors:
            walk(c, depth + 1)
    walk(tn, 0)
    return best[1]


def net_k1():
    """two 64 x 42 x 64 GEMM-like pairs with mixed extents (K1 DMMA both ways), a dim-1 leg, an open leg of 3"""
    rng = np.random.default_rng(101)
    dim = {0: 64, 1: 6, 2: 7, 3: 64, 4: 1, 5: 5, 6: 3}
    legs = [[0, 1, 2], [2, 1, 3, 4], [0, 5], [3, 5, 6, 4]]
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    tn = Tensor.new_composite(make_leaves(legs, dim, rng))
    return Net("k1_dmma", tn, ContractionPath.simple([(0, 1), (0, 2), (0, 3)]), routes={"k1_dmma", "k0"},
               sliced=[[1], [1, 5]])


def net_k2():
    """an outer product (no shared leg) of a (7,5,3,3) and a (4,4,3) leaf: a 15120-entry intermediate with a big side of
    7*5*3*4*4*3 that K2 streams against a 3x3 and a (3, 3, 1, 2) leaf (big side not a power of two); the closing pair
    contracts K = 7560 with a rank-8 leaf onto 4 outputs (K0 split-K); result rank 1"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    rng = np.random.default_rng(102)
    dim = {0: 7, 1: 5, 2: 3, 3: 3, 4: 4, 5: 4, 6: 3, 7: 3, 8: 3, 9: 1, 10: 2}
    legs = [[0, 1, 2, 3], [4, 5, 6], [3, 7], [8, 6, 9, 10], [1, 7, 0, 5, 10, 8, 9, 2]]
    tn = Tensor.new_composite(make_leaves(legs, dim, rng))
    return Net("k2_odd_outer", tn, ContractionPath.simple([(0, 1), (0, 2), (0, 3), (0, 4)]),
               routes={"k2", "k0_splitk"}, sliced=[[3], [1, 2], [2, 1, 0]])


def net_int8():
    """A (7,5,4 | 3,7,7) x B (7,3,7 | 5,5,6): M = 140, K = 147, N = 150; the closing pair contracts K = 21000 to a scalar.
    Under set_tcgen05_threshold(1, 128) the forward pair and the adjoints of both leaves take the int8 engine"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    rng = np.random.default_rng(103)
    dim = {0: 7, 1: 5, 2: 4, 3: 3, 4: 7, 5: 7, 6: 5, 7: 5, 8: 6}
    legs = [[0, 1, 2, 3, 4, 5], [5, 3, 4, 6, 7, 8], [7, 0, 8, 1, 2, 6]]
    tn = Tensor.new_composite(make_leaves(legs, dim, rng))
    return Net("int8_engine", tn, ContractionPath.simple([(0, 1), (0, 2)]), int8=True,
               routes={"k1_tcgen05", "k0_splitk"}, sliced=[[3], [5, 3]])


def k3_legs(rank, dims):
    """a rank-`rank` leaf X whose odd legs meet O in reverse order and whose even legs meet P in a shuffled order: X's
    adjoint comes out as (O's legs) ++ (P's side), and no two neighbouring legs of X are neighbours there"""
    X = list(range(rank))
    odd = [l for l in X if l % 2][::-1]
    even = [l for l in X if not l % 2]
    even = even[1::2] + even[0::2]
    dim = dict(zip(X, dims))
    dim[100], dim[101] = 3, 2
    return [X, odd + [100], even + [101]], dim


def net_k3_flat():
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    rng = np.random.default_rng(104)
    legs, dim = k3_legs(12, [2, 3, 2, 2, 3, 2, 2, 2, 2, 3, 2, 2])
    tn = Tensor.new_composite(make_leaves(legs, dim, rng))
    return Net("k3_rank12", tn, ContractionPath.simple([(0, 1), (0, 2)]), routes={"permute"},
               sliced=[[1], [4, 1], [1, 2, 4]])


def net_k3_nested():
    """the rank-10 X inside a composite with P, O alone in a single-leaf composite, a rank-0 leaf at the top level"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    rng = np.random.default_rng(105)
    legs, dim = k3_legs(10, [3, 2, 2, 5, 2, 2, 3, 2, 2, 2])
    lv = make_leaves(legs + [[]], dim, rng)
    tn = Tensor.new_composite([Tensor.new_composite([lv[0], lv[2]]), Tensor.new_composite([lv[1]]), lv[3]])
    path = ContractionPath({0: ContractionPath.simple([(0, 1)]), 1: ContractionPath.simple([])}, [(0, 1), (0, 2)])
    return Net("k3_rank10_nested", tn, path, routes={"permute"}, deep=0, sliced=[[6], [3, 0]])


def net_sliced_mixed():
    """a leaf with the sliced legs 5 and 3 in the opposite order to the sliced-leg list [3, 2, 5], a sliced leg next to a
    dim-1 leg, a leaf whose only legs are sliced, a (3, 5) leaf, a rank-3 result"""
    from tnc_b200.tensornetwork import Tensor
    rng = np.random.default_rng(106)
    dim = {0: 3, 1: 2, 2: 5, 3: 3, 4: 7, 5: 1, 6: 2, 7: 5, 8: 3, 9: 2}
    dim.update({10: 2, 11: 3, 12: 5})
    # leaf 0 carries the sliced legs 2 and 0 in that order; leaf 1 has the dim-1 leg 5 next to the sliced leg 0; leaf 2
    # carries only sliced legs; leaf 5 is (3, 5); the open legs 10, 11, 12 sit on leaves 3, 6 and 1
    legs = [[4, 2, 0, 9], [5, 0, 1, 12], [1, 2], [6, 4, 7, 10], [8, 6, 5], [3, 7], [3, 9, 8, 11]]
    lv = make_leaves(legs, dim, rng)
    tn = Tensor.new_composite(lv)
    path = tree_path(tn, rng)
    return Net("sliced_mixed", tn, path, sliced=[[0], [2, 1], [0, 1, 2]], routes={"k0"})


def net_sliced_mixed_nested():
    """the same structure in three composites, one of them nested two deep"""
    from tnc_b200.tensornetwork import Tensor
    base = net_sliced_mixed()
    tn = build_tree(base.leaves, [[0, [1, 2]], [3, 4], [5], 6])
    rng = np.random.default_rng(107)
    return Net("sliced_mixed_nested", tn, tree_path(tn, rng, "random"), sliced=[[0], [2, 1], [0, 1, 2]],
               routes={"k0"}, deep=deepest_leaf(tn))


def net_disconnected():
    """two components joined by an outer product, rank-0 leaves, a rank-5 result over both components"""
    return random_net("disconnected", 201, 8, 2, 5, components=2, n_rank0=2)


def corpus_specs():
    W = [0.1, 0.35, 0.3, 0.15, 0.1]
    specs = [net_k1, net_k2, net_int8, net_k3_flat, net_k3_nested, net_sliced_mixed, net_sliced_mixed_nested,
             net_disconnected]
    specs += [functools.partial(random_net, f"flat_greedy_{s}", s, n, e, o, weights=W)
              for s, n, e, o in ((301, 6, 2, 0), (302, 8, 3, 1), (303, 9, 2, 2), (304, 7, 4, 3), (305, 10, 3, 4))]
    specs += [functools.partial(random_net, f"flat_random_{s}", s, n, e, o, kind="random", weights=W)
              for s, n, e, o in ((311, 7, 2, 0), (312, 8, 2, 2), (313, 9, 3, 6))]
    specs += [functools.partial(random_net, f"partition_{s}", s, n, e, o, partition=p, weights=W)
              for s, n, e, o, p in ((321, 8, 3, 1, [0, 1, 0, 2, 1, 2, 0, 1]), (322, 9, 2, 3, [1, 1, 0, 0, 2, 3, 2, 3, 3]),
                                    (323, 6, 2, 0, [0, 1, 1, 1, 1, 1]))]
    specs += [functools.partial(random_net, f"nested_{s}", s, n, e, o, groups=g, kind=k, weights=W)
              for s, n, e, o, g, k in ((331, 8, 3, 2, [[0, 1, [2, 3]], [4], 5, [6, 7]], "greedy"),
                                       (332, 9, 2, 1, [[[0, 1], 2], [[3], [4, 5]], [6, 7, 8]], "random"),
                                       (333, 7, 3, 4, [[0, 1, 2, 3], [4, 5, 6]], "greedy"),
                                       (334, 10, 2, 0, [[0, 1], [2, 3], [4, 5, 6], [7, 8, 9]], "random"),
                                       (335, 6, 2, 3, [0, [1], [2, 3], [4, 5]], "random"))]
    return specs


@functools.lru_cache(maxsize=None)
def corpus():
    return {n.name: n for n in (f() for f in corpus_specs())}


def names():
    return ["k1_dmma", "k2_odd_outer", "int8_engine", "k3_rank12", "k3_rank10_nested", "sliced_mixed",
            "sliced_mixed_nested", "disconnected", "flat_greedy_301", "flat_greedy_302", "flat_greedy_303",
            "flat_greedy_304", "flat_greedy_305", "flat_random_311", "flat_random_312", "flat_random_313",
            "partition_321", "partition_322", "partition_323", "nested_331", "nested_332", "nested_333", "nested_334",
            "nested_335"]


def get(name):
    return corpus()[name]


NAMES = ["k1_dmma", "k2_odd_outer", "int8_engine", "k3_rank12", "k3_rank10_nested", "sliced_mixed",
         "sliced_mixed_nested", "disconnected", "flat_greedy_301", "flat_greedy_302", "flat_greedy_303", "flat_greedy_304",
         "flat_greedy_305", "flat_random_311", "flat_random_312", "flat_random_313", "partition_321", "partition_322",
         "partition_323", "nested_331", "nested_332", "nested_333", "nested_334", "nested_335"]


def nrng(name, salt=0):
    """a generator seeded by the network's name: every test draws the same seeds and tangents on every run"""
    import zlib
    return np.random.default_rng(zlib.crc32(name.encode()) + salt)


def with_payloads(t, xs):
    """the tree t with its leaves' payloads replaced by xs (depth-first)"""
    from tnc_b200.tensornetwork import Tensor
    it = iter(xs)

    def walk(u):
        if not u.tensors:
            return matrix_leaf(u.legs, u.bond_dims, next(it))
        return Tensor.new_composite([walk(c) for c in u.tensors])
    return walk(t)


def with_extent(net, d):
    """net with every extent set to d and fresh payloads (same seeds): the equal-extent twin of a general network"""
    from tnc_b200.tensornetwork import Tensor
    rng = nrng(net.name, 7)

    def walk(u):
        if not u.tensors:
            shape = [d] * len(u.legs)
            return matrix_leaf(u.legs, shape, crandn(rng, shape))
        return Tensor.new_composite([walk(c) for c in u.tensors])
    return Net(net.name + f"_all{d}", walk(net.tn), net.path, sliced=net.sliced, deep=net.deep)


def result_dims(net):
    return tuple(ref_value(net)[1].shape)


# ================================================================================================================
# 2. the reference
# ================================================================================================================
def ttgt(a_legs, A, b_legs, B):
    """C[(b\\a) ++ (a\\b)] = sum over the shared legs: transpose, reshape, one GEMM, reshape"""
    import torch
    shared = [l for l in a_legs if l in b_legs]
    am = [l for l in a_legs if l not in b_legs]
    bn = [l for l in b_legs if l not in a_legs]
    dim = dict(zip(a_legs, A.shape)) | dict(zip(b_legs, B.shape))
    size = lambda ls: int(np.prod([dim[l] for l in ls], dtype=np.int64))
    At = A.permute([a_legs.index(l) for l in shared + am]).reshape(size(shared), size(am))
    Bt = B.permute([b_legs.index(l) for l in bn + shared]).reshape(size(bn), size(shared))
    return bn + am, torch.matmul(Bt, At).reshape([dim[l] for l in bn + am])


def replay(tn, path, xs):
    """(legs, R): `tn` contracted along the replace-left `path`, nested or flat, in torch; xs = the leaves' tensors in
    depth-first order"""
    it = iter(xs)

    def walk(t, p):
        if not t.tensors:
            return list(t.legs), next(it)
        slots = [walk(c, p.nested.get(i) if c.tensors else None) for i, c in enumerate(t.tensors)]
        for i, j in p.toplevel:
            slots[i] = ttgt(*slots[i], *slots[j])
            slots[j] = None
        return next(s for s in slots if s is not None)
    return walk(tn, path)


def T(x):
    import torch
    return torch.tensor(np.asarray(x, dtype=np.complex128))


def ref_value(net, xs=None):
    legs, R = replay(net.tn, net.path, [T(x) for x in (net.xs if xs is None else xs)])
    return legs, R.numpy()


def ref_grads(net, seed, xs=None, tn=None):
    """(R, [G_l for every leaf]) with G_l = sum_r seed[r] dR[r]/dX_l: torch returns conj of that for grad_outputs =
    conj(seed)"""
    import torch
    X = [T(x).requires_grad_() for x in (net.xs if xs is None else xs)]
    _, R = replay(net.tn if tn is None else tn, net.path, X)
    gs = torch.autograd.grad(R, X, grad_outputs=T(seed).conj())
    return R.detach().numpy(), [g.conj().resolve_conj().numpy() for g in gs]


def tangent_list(net, tans):
    return [np.asarray(tans[i], dtype=np.complex128) if i in tans else np.zeros_like(x) for i, x in enumerate(net.xs)]


def ref_jvp(net, tans):
    """(R, Ṙ): torch.func.jvp of the replay; tans = {leaf: Ẋ}, the other leaves have zero tangent"""
    import torch
    f = lambda *ys: replay(net.tn, net.path, ys)[1]
    R, Rd = torch.func.jvp(f, tuple(T(x) for x in net.xs), tuple(T(t) for t in tangent_list(net, tans)))
    return R.numpy(), Rd.numpy()


def ref_hvp(net, tans, seed, seed_tan):
    """([G_l], [Ġ_l]): jvp of the conjugated vjp of the replay, along the leaf tangents and the seed tangent"""
    import torch
    f = lambda *ys: replay(net.tn, net.path, ys)[1]
    n = len(net.xs)

    def grads(*args):
        _, back = torch.func.vjp(f, *args[:n])
        return tuple(g.conj() for g in back(args[n].conj()))
    G, Gd = torch.func.jvp(grads, tuple(T(x) for x in net.xs) + (T(seed),),
                           tuple(T(t) for t in tangent_list(net, tans)) + (T(seed_tan),))
    return [g.resolve_conj().numpy() for g in G], [g.resolve_conj().numpy() for g in Gd]


def mixed_digits(q, ext):
    """slice q as the row-major digit vector over the sliced legs, last leg fastest"""
    out = []
    for e in reversed(ext):
        out.append(q % e)
        q //= e
    return out[::-1]


def bit_digits(q, ext):
    """the planted fault: digit k taken as a bit of q, k counting from the last leg"""
    return [(q >> (len(ext) - 1 - k)) & 1 for k in range(len(ext))]


def strip(t, sl):
    """the tree t with the legs sl removed from every leaf (the structure every slice shares)"""
    from tnc_b200.tensornetwork import Tensor
    if not t.tensors:
        keep = [(l, d) for l, d in zip(t.legs, t.bond_dims) if l not in sl]
        return Tensor([l for l, _ in keep], [d for _, d in keep])
    return Tensor.new_composite([strip(c, sl) for c in t.tensors])


def ref_sliced(net, legs, slices, seed, digits=mixed_digits, xs=None):
    """(R, [G_l], [touched_l]) summed over exactly `slices` of the legs `legs`: each slice cut from the full leaves with
    numpy indexing, replayed along the path, its gradients embedded back into the full leaf shapes; touched_l marks
    the entries of leaf l that some requested slice reaches"""
    xs = net.xs if xs is None else xs
    ext = [net.dim[l] for l in legs]
    skel = strip(net.tn, set(legs))
    R = 0
    G = [np.zeros_like(x) for x in xs]
    touched = [np.zeros(x.shape, dtype=bool) for x in xs]
    for q in slices:
        val = dict(zip(legs, digits(q, ext)))
        idx = [tuple(val.get(l, slice(None)) for l in t.legs) for t in net.leaves]
        r, g = ref_grads(net, seed, [x[i] for x, i in zip(xs, idx)], tn=skel)
        R = R + r
        for l, i in enumerate(idx):
            G[l][i] += g[l]
            touched[l][i] = True
    return R, G, touched


def rel_err(got, ref):
    """max |got - ref| in units of the largest reference entry"""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    unit = np.abs(ref).max() if ref.size else 0.0
    d = np.abs(got - ref).max() if ref.size else 0.0
    return d / unit if unit > 0 else d


WORST = {}


def check(kind, got, ref, tau, what=""):
    """assert rel_err <= tau and keep the worst error per plan kind"""
    e = rel_err(got, ref)
    WORST[kind] = max(WORST.get(kind, 0.0), e)
    assert e <= tau, (kind, what, e, tau)
    return e


def tau_of(net):
    """TAU on FP64 routes; with the int8 engine its bound at the longest contraction length it takes (K = 150) in units
    of max|a| max|b|, times 256 for the closing K = 21000 contraction it feeds (sqrt(21000) = 145) and the operands' spread"""
    if not net.int8:
        return TAU
    import tnc_b200 as tb
    return TAU + 256 * tb.tcgen05_bound(150)["bound"]


def einsum_value(net):
    """the whole network by a path-independent np.einsum, output legs in the reference's order"""
    legs, _ = ref_value(net)
    letters = {}
    sym = lambda ls: "".join(letters.setdefault(l, chr(ord("A") + len(letters) + (6 if len(letters) >= 26 else 0)))
                             for l in ls)
    ops = ",".join(sym(t.legs) for t in net.leaves)
    return np.einsum(ops + "->" + sym(legs), *net.xs, optimize="greedy")


# ================================================================================================================
# 1. and 2. on the host
# ================================================================================================================
def test_corpus_invariants():
    """the generator's promises: names, extents, ranks, result ranks, every leg on at most two leaves, nested and flat
    paths, per-leaf scales, intermediates small enough for the host reference"""
    c = corpus()
    assert sorted(c) == sorted(NAMES)
    ranks, extents, res_ranks, kinds, scales = set(), set(), set(), set(), []
    for net in c.values():
        count = {}
        for t in net.leaves:
            ranks.add(len(t.legs))
            extents.update(t.bond_dims)
            for l in t.legs:
                count[l] = count.get(l, 0) + 1
        assert max(count.values()) <= 2, net.name
        res_ranks.add(len(ext_legs(net.tn)))
        kinds.add("flat" if net.flat else "nested")
        peak = 0
        for *_, al, ad, bl, bd in forward_steps(net):
            peak = max(peak, int(np.prod(out_legs(al, ad, bl, bd)[1], dtype=np.int64)))
        assert peak <= 1 << 15, (net.name, peak)
        spread = [np.abs(x).max() for x in net.xs]
        scales.append(max(spread) / min(spread))
        for sl in net.sliced:
            assert all(count.get(l) == 2 for l in sl), (net.name, sl)      # bonds, never open legs
    assert set(range(0, 9)) <= ranks and {10, 12} <= ranks, ranks
    assert set(POOL) <= extents and max(extents) >= 64, extents
    assert {0, 1, 2, 3, 4, 5, 6} <= res_ranks, res_ranks
    assert kinds == {"flat", "nested"}
    assert max(scales) > 2.0 ** 12, max(scales)                           # leaves scaled 2^-8 .. 2^8 apart
    sl = {tuple(get(n).dim[l] for l in s) for n in NAMES for s in get(n).sliced}
    assert {(3,), (5, 2), (3, 2, 5)} <= sl, sl
    # the hand-built slicing cases: a leaf with two sliced legs in the opposite order, a sliced leg next to a dim-1 leg
    sm = get("sliced_mixed")
    assert sm.leaves[0].legs.index(2) < sm.leaves[0].legs.index(0)
    assert sm.leaves[1].legs[:2] == [5, 0] and sm.dim[5] == 1
    # nested: single-leaf composites, two levels of nesting, a leaf among composites, partition_tensor_network
    assert any(len(c.tensors) == 1 for n in NAMES for c in get(n).tn.tensors if c.tensors)
    assert any(g.tensors for n in NAMES for c in get(n).tn.tensors for g in c.tensors)
    assert any(not c.tensors for n in NAMES if not get(n).flat for c in get(n).tn.tensors)


def out_legs(al, ad, bl, bd):
    """legs and dims of contract(a, b): (b \\ a) ++ (a \\ b)"""
    return ([l for l in bl if l not in al] + [l for l in al if l not in bl],
            [d for l, d in zip(bl, bd) if l not in al] + [d for l, d in zip(al, ad) if l not in bl])


def forward_steps(net):
    """(slot of a, slot of b, a legs, a dims, b legs, b dims) of every forward step in build()'s order: nested children
    first in child order, depth first, then the level's own pairs; slots ("leaf", i) / ("step", q)"""
    steps, counter = [], [0]

    def walk(t, p):
        if not t.tensors:
            counter[0] += 1
            return ("leaf", counter[0] - 1), list(t.legs), list(t.bond_dims)
        slots = [walk(c, p.nested.get(i) if c.tensors else None) for i, c in enumerate(t.tensors)]
        for i, j in p.toplevel:
            (sa, al, ad), (sb, bl, bd) = slots[i], slots[j]
            steps.append((sa, sb, al, ad, bl, bd))
            slots[i], slots[j] = (("step", len(steps) - 1),) + tuple(out_legs(al, ad, bl, bd)), None
        return next(s for s in slots if s is not None)
    walk(net.tn, net.path)
    return steps


def backward_pairs(steps):
    """(C-bar legs, C-bar dims, other legs, other dims, operand slot) of every backward pair with every leaf requested,
    in build_backward's order: the steps from the root, operand a then operand b; the root's adjoint is the seed"""
    adj = {("step", len(steps) - 1): out_legs(*steps[-1][2:])}
    pairs = []
    for q in range(len(steps) - 1, -1, -1):
        a, b, al, ad, bl, bd = steps[q]
        gl, gd = adj.pop(("step", q))
        for x, (ol, od) in ((a, (bl, bd)), (b, (al, ad))):
            pairs.append((gl, gd, ol, od, x))
            adj[x] = tuple(out_legs(gl, gd, ol, od))
    return pairs


def kernel_class(al, ad, bl, bd):
    from tnc_b200._lib import lib, u64_array
    return lib().tncb_pair_kernel_class(len(al), u64_array(al), u64_array(ad), len(bl), u64_array(bl), u64_array(bd))


def mnk(al, ad, bl, bd):
    M = int(np.prod([d for l, d in zip(al, ad) if l not in bl], dtype=np.int64))
    N = int(np.prod([d for l, d in zip(bl, bd) if l not in al], dtype=np.int64))
    K = int(np.prod([d for l, d in zip(al, ad) if l in bl], dtype=np.int64))
    return M, N, K


def k2_big_dims(al, ad, bl, bd):
    """the extents of the side K2 streams (plan_pair: a's free legs if N is the small side, else b's)"""
    M, N, K = mnk(al, ad, bl, bd)
    if N <= 16 and N * K <= 256 and M >= 4096:
        return [d for l, d in zip(al, ad) if l not in bl]
    return [d for l, d in zip(bl, bd) if l not in al]


def gather_groups(leaf_legs, leaf_dims, adj_legs, adj_dims):
    """fused leg groups of a leaf's gradient gather (build_gather): the leaf's legs in its order, strides in the adjoint"""
    st, s = {}, 1
    for l, d in zip(reversed(adj_legs), reversed(adj_dims)):
        st[l], s = s, s * d
    groups = []
    for l, d in zip(leaf_legs, leaf_dims):
        if d == 1:
            continue
        if groups and groups[-1] == st[l] * d:
            groups[-1] = st[l]
            continue
        groups.append(st[l])
    return len(groups)


def host_plan_info(net, kind):
    from tnc_b200._lib import lib
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(net.tn), m.path(net.path)
    h = C.c_void_p()
    rc = (lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)) if kind == "plain" else
          lib().tncb_plan_create_vjp(None, C.byref(ct), C.byref(cp), None, C.byref(h)))
    assert rc == 0, lib().tncb_last_error()
    try:
        n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
        fl, by = C.c_double(), C.c_double()
        assert lib().tncb_plan_info(h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
        return n.value, fl.value
    finally:
        lib().tncb_plan_destroy(h)


def test_route_inventory(built_lib):
    """forward and restated backward pairs: counts and flops equal host-only plans'; across the corpus they reach K0, K1
    and K2 (one K2 pair with a big side that is not a power of two), and leaf adjoints need more than 8 fused groups"""
    classes = {0: 0, 1: 0, 2: 0}
    odd_k2, many_groups = [], []
    for name in NAMES:
        net = get(name)
        steps = forward_steps(net)
        bw = backward_pairs(steps)
        flops = 0.0
        for pair in [s[2:] for s in steps] + [p[:4] for p in bw]:
            cls = kernel_class(*pair)
            classes[cls] += 1
            M, N, K = mnk(*pair)
            flops += 8.0 * M * N * K
            if cls == 2 and any(d & (d - 1) for d in k2_big_dims(*pair)):
                odd_k2.append(name)
        assert host_plan_info(net, "plain") == (len(steps), pytest.approx(sum(8.0 * np.prod(mnk(*s[2:]), dtype=np.float64)
                                                                              for s in steps), rel=1e-12)), name
        assert host_plan_info(net, "vjp") == (len(steps) + len(bw), pytest.approx(flops, rel=1e-12)), name
        for gl, gd, ol, od, x in bw:
            if x[0] == "leaf":
                al, ad = out_legs(gl, gd, ol, od)
                leaf = net.leaves[x[1]]
                if gather_groups(leaf.legs, leaf.bond_dims, al, ad) > 8:
                    many_groups.append((name, x[1]))
    assert all(classes[c] > 0 for c in (0, 1, 2)), classes
    assert "k2_odd_outer" in odd_k2, odd_k2
    assert ("k3_rank12", 0) in many_groups and ("k3_rank10_nested", 0) in many_groups, many_groups


@pytest.mark.parametrize("name", NAMES)
def test_reference_against_einsum(name):
    """the replay of the path equals a path-independent einsum of the whole network"""
    net = get(name)
    _, R = ref_value(net)
    assert rel_err(R, einsum_value(net)) <= 1e-13, name


@pytest.mark.parametrize("name", [n for n in NAMES if get(n).sliced])
def test_sliced_reference_folds_to_unsliced(name):
    """the sliced reference summed over every slice equals the unsliced reference, value and every leaf"""
    net = get(name)
    rng = nrng(name, 1)
    seed = crandn(rng, result_dims(net))
    R, G = ref_grads(net, seed)
    for legs in net.sliced:
        n = int(np.prod([net.dim[l] for l in legs]))
        Rs, Gs, touched = ref_sliced(net, legs, range(n), seed)
        assert rel_err(Rs, R) <= 1e-13, (name, legs)
        for l in range(len(G)):
            assert touched[l].all()
            assert rel_err(Gs[l], G[l]) <= 1e-13, (name, legs, l)


# ================================================================================================================
# 4. the comparator against planted faults (host)
# ================================================================================================================
def wrong_extents(G):
    """the planted fault: a leaf gradient addressed with the extents of its legs in reverse order (a (3, 5) leaf read as
    rows of 3), the error of code that reads the extent of the wrong leg"""
    d = G.shape
    rev = d[::-1]
    st = [int(np.prod(rev[k + 1:], dtype=np.int64)) for k in range(len(d))]
    idx = sum(i * s for i, s in zip(np.indices(d), st))
    return G.reshape(-1)[idx]


def test_comparator_rejects_planted_faults():
    net = get("sliced_mixed")
    seed = crandn(nrng(net.name, 2), result_dims(net))
    twin = with_extent(net, 2)
    seed2 = crandn(nrng(net.name, 3), result_dims(twin))
    _, G = ref_grads(net, seed)
    _, G2 = ref_grads(twin, seed2)
    # a (3, 5) gradient read with the extents of (5, 3): rejected; on the all-2 twin the same code is right
    assert G[5].shape == (3, 5)
    assert rel_err(wrong_extents(G[5]), G[5]) > 1e-3
    assert rel_err(wrong_extents(G2[5]), G2[5]) == 0.0
    # slice digits taken as bits: at extents (3, 2, 5) the full range and the single slice with digits (1, 1, 1) fail
    legs = [0, 1, 2]
    assert [net.dim[l] for l in legs] == [3, 2, 5]
    q = 1 * 10 + 1 * 5 + 1
    assert mixed_digits(q, [3, 2, 5]) == [1, 1, 1]
    for sl, sl2 in ((range(30), range(8)), ([q], [7])):                   # q = 7: digits (1, 1, 1) at extents 2
        R, Gs, _ = ref_sliced(net, legs, sl, seed)
        Rb, Gb, _ = ref_sliced(net, legs, sl, seed, digits=bit_digits)
        assert rel_err(Rb, R) > 1e-3 and max(rel_err(a, b) for a, b in zip(Gb, Gs)) > 1e-3, sl
        R2, G2s, _ = ref_sliced(twin, legs, sl2, seed2)
        Rb2, G2b, _ = ref_sliced(twin, legs, sl2, seed2, digits=bit_digits)
        assert rel_err(Rb2, R2) == 0.0 and all(rel_err(a, b) == 0.0 for a, b in zip(G2b, G2s))
    # 1e-9 relative change of one entry of the smallest leaf's gradient: rejected in per-leaf units on every network;
    # in the units of the largest gradient entry over all leaves (the older small-scale files) it slips through on some
    slipped = []
    for name in NAMES:
        n = get(name)
        _, G = ref_grads(n, crandn(nrng(name, 4), result_dims(n)))
        small = min(range(len(G)), key=lambda l: (G[l].size, l))
        bad = G[small].copy()
        k = np.unravel_index(np.abs(bad).argmax(), bad.shape)
        bad[k] *= 1 + 1e-9
        assert rel_err(bad, G[small]) > TAU, name
        gmax = max(np.abs(g).max() for g in G)
        if np.abs(bad - G[small]).max() <= TAU * gmax:
            slipped.append(name)
    assert slipped, "no network shows the global unit's blind spot"


# ================================================================================================================
# 3. every plan kind on the GPU
# ================================================================================================================
@pytest.fixture(scope="module")
def ctxs(built_lib):
    """the default context, and one that routes every pair with M, N >= 128 and K >= 128 to the int8 engine"""
    import tnc_b200 as tb
    c, c8 = tb.Context(0), tb.Context(0)
    c8.set_tcgen05_threshold(1, 128)
    yield c, c8
    c.close()
    c8.close()


def ctx_of(ctxs, net):
    return ctxs[1] if net.int8 else ctxs[0]


ENGINES = {}


def counted(c, fn):
    """(fn(), the engine counts of that call); the counts are also summed over the corpus for the report"""
    c.reset_stats()
    res = fn()
    c.synchronize()
    ec = c.engine_counts()
    for k in COUNTERS:
        ENGINES[k] = ENGINES.get(k, 0) + ec[k]
    return res, ec


def instances(net, n):
    """n payload sets of net: the network's own, then fresh random ones"""
    rng = nrng(net.name, 10)
    return [net.xs] + [[crandn(rng, x.shape) * 2.0 ** int(rng.integers(-8, 9)) for x in net.xs] for _ in range(n - 1)]


def subset(net):
    """a random subset of the leaves that keeps the deep leaf and drops at least one leaf"""
    rng = nrng(net.name, 11)
    n = len(net.leaves)
    pick = set(int(i) for i in rng.choice(n, max(1, n // 2), replace=False)) | {net.deep}
    if len(pick) == n:
        pick.discard(min(pick - {net.deep}))
    return sorted(pick)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_forward(ctxs, name, monkeypatch):
    """contract_tensor_network twice (the second sighting runs the cached plan), stage + run, execute, and the
    pair-by-pair executor, against the reference; the pair-by-pair executor's engine counts hold the routes the
    network was built for"""
    from tnc_b200.tensornetwork import NetworkPlan, contract_tensor_network
    net = get(name)
    c = ctx_of(ctxs, net)
    legs, R = ref_value(net)
    tau = tau_of(net)
    for k in range(2):
        r = contract_tensor_network(net.tn, net.path, ctx=c)
        assert r.legs == legs
        check("forward", r.to_numpy(), R, tau, f"direct {k}")
    plan = NetworkPlan(net.tn, net.path, ctx=c)
    plan.stage(net.tn)
    check("forward", plan.run().to_numpy(), R, tau, "run")
    check("forward", plan.execute(net.tn).to_numpy(), R, tau, "execute")
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    pbp = NetworkPlan(net.tn, net.path, ctx=c)
    monkeypatch.delenv("TNCB_NO_STATIC")
    r, ec = counted(c, lambda: pbp.execute(net.tn))
    check("forward", r.to_numpy(), R, tau, "pair by pair")
    fwd_routes = {"k1_dmma": ("k1_dmma",), "k2_odd_outer": ("k2", "k0_splitk"),
                  "int8_engine": ("k1_tcgen05", "k0_splitk")}.get(name, ())
    for route in fwd_routes:
        assert ec[route] > 0, (name, route, ec)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_batched_forward(ctxs, name):
    """run_batch over instances with different payloads, every row against its own reference; run_slices(i, n) for
    each instance and run_slices(0, 1) for their sum"""
    from tnc_b200.tensornetwork import NetworkPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    n = 3
    xss = instances(net, n)
    refs = [ref_value(net, xs)[1] for xs in xss]
    nets = [with_payloads(net.tn, xs) for xs in xss]
    plan = NetworkPlan(nets[0], net.path, ctx=c)
    plan.stage_slices(nets)
    legs, rows = plan.run_batch(0, n)
    assert legs == ref_value(net)[0]
    rows = rows.to_numpy()
    for i in range(n):
        check("batched forward", rows[i], refs[i], tau_of(net), f"row {i}")
        check("batched forward", plan.run_slices(i, n).to_numpy(), refs[i], tau_of(net), f"run_slices({i}, {n})")
    check("batched forward", plan.run_slices(0, 1).to_numpy(), sum(refs), tau_of(net), "sum")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gradients(ctxs, name, monkeypatch):
    """gradient plans with a random seed of the result's shape, wrt every leaf, a random subset and the deep leaf; every
    G_l in units of its own largest entry; the routes of the forward pass and the backward pass"""
    from tnc_b200.tensornetwork import NetworkPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    seed = crandn(nrng(name, 12), result_dims(net))
    R, G = ref_grads(net, seed)
    tau = tau_of(net)
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    pbp = NetworkPlan(net.tn, net.path, ctx=c)
    monkeypatch.delenv("TNCB_NO_STATIC")
    _, routes = counted(c, lambda: pbp.execute(net.tn))
    for wrt in (None, subset(net), [net.deep]):
        plan = NetworkPlan.for_gradients(net.tn, net.path, wrt, ctx=c)
        plan.stage(net.tn)
        check("gradient", plan.run().to_numpy(), R, tau, "value")
        g, ec = counted(c, lambda: plan.vjp(seed))
        if wrt is None:
            routes = {k: routes[k] + ec[k] for k in routes}
        assert sorted(g) == (list(range(len(G))) if wrt is None else sorted(wrt)), (name, wrt)
        for l in g:
            check("gradient", g[l], G[l], tau, f"wrt {wrt} leaf {l}")
    for route in net.routes:
        assert routes[route] > 0, (name, route, routes)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_batched_gradients(ctxs, name):
    """vjp_batch over instances with different payloads and seeds: values and rows against their references, the sum
    equal bit for bit to the left fold of the rows"""
    from tnc_b200.tensornetwork import NetworkPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    n = 3
    xss = instances(net, n)
    seeds = crandn(nrng(name, 13), (n,) + result_dims(net))
    plan = NetworkPlan.for_gradients(net.tn, net.path, ctx=c)
    plan.stage_batch([with_payloads(net.tn, xs) for xs in xss])
    _, vals, rows, total = plan.vjp_batch(0, n, seeds, rows=True, sum=True)
    for i in range(n):
        R, G = ref_grads(net, seeds[i], xss[i])
        check("batched gradient", vals[i], R, tau_of(net), f"value {i}")
        for l in range(len(G)):
            check("batched gradient", rows[l][i], G[l], tau_of(net), f"row {i} leaf {l}")
    for l in rows:
        fold = rows[l][0].copy()
        for i in range(1, n):
            fold = fold + rows[l][i]
        assert np.array_equal(total[l], fold), (name, l)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_tangents(ctxs, name):
    """jvp along random tangents of a subset of the leaves; jvp_batch over P directions of one network staged as
    stride-0 instances, every row against the reference of its direction"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    rng = nrng(name, 14)
    wrt = subset(net)
    plan = NetworkPlan.for_tangents(net.tn, net.path, wrt, ctx=c)
    plan.stage(net.tn)
    tans = {l: crandn(rng, net.xs[l].shape) for l in wrt}
    R, Rd = ref_jvp(net, tans)
    v, t = plan.jvp(tans)
    check("tangent", v.to_numpy(), R, tau_of(net), "value")
    check("tangent", t, Rd, tau_of(net), "tangent")
    P = 3
    rows = {l: crandn(rng, (P,) + net.xs[l].shape) for l in wrt}
    first = wrt[0]
    plan.stage_instances(net.tn, {first: torch.from_numpy(net.xs[first]).cuda()}, P)
    _, vals, trows = plan.jvp_batch(0, P, rows)
    for p in range(P):
        R, Rd = ref_jvp(net, {l: x[p] for l, x in rows.items()})
        check("batched tangent", vals[p], R, tau_of(net), f"value {p}")
        check("batched tangent", trows[p], Rd, tau_of(net), f"direction {p}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_hvp(ctxs, name):
    """a Hessian-vector plan on a subset of the leaves with a random seed and a non-zero seed tangent: R, Ṙ, G and Ġ"""
    from tnc_b200.tensornetwork import NetworkPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    rng = nrng(name, 15)
    wrt = subset(net)
    dims = result_dims(net)
    seed, seed_tan = crandn(rng, dims), crandn(rng, dims)
    tans = {l: crandn(rng, net.xs[l].shape) for l in wrt}
    plan = NetworkPlan.for_hvp(net.tn, net.path, wrt, ctx=c)
    plan.stage(net.tn)
    value, tangent, g, dg = plan.hvp(tans, seed, seed_tan)
    R, Rd = ref_jvp(net, tans)
    G, Gd = ref_hvp(net, tans, seed, seed_tan)
    tau = tau_of(net)
    check("hvp", value, R, tau, "value")
    check("hvp", tangent, Rd, tau, "tangent")
    assert sorted(g) == sorted(dg) == wrt
    for l in wrt:
        check("hvp", g[l], G[l], tau, f"G {l}")
        check("hvp", dg[l], Gd[l], tau, f"Ġ {l}")


SLICED = [(n, k) for n in NAMES for k in range(len(get(n).sliced))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,k", SLICED)
def test_sliced_gradients(ctxs, name, k):
    """a sliced gradient plan on mixed-radix legs: the full range, single slices whose digits are all non-zero, a
    (rank, world) sub-range, each against a reference of exactly those slices, with every entry outside their sub-blocks
    exactly 0; on flat networks the forward SlicedPlan on the same legs"""
    from tnc_b200.contractionpath.slicing import SlicedPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    legs = net.sliced[k]
    ext = [net.dim[l] for l in legs]
    n = int(np.prod(ext))
    seed = crandn(nrng(name, 16 + k), result_dims(net))
    tau = tau_of(net)
    sp = SlicedPlan.for_gradients(net.tn, net.path, legs, ctx=c)
    sp.stage(net.tn)
    ones = sum(int(np.prod(ext[i + 1:])) for i in range(len(ext)))          # the slice with every digit 1
    world = 3 if n >= 3 else 2
    for rank, w in ((0, 1), (ones, n), (n - 1, n), (1, world)):
        sl = list(range(rank, n, w))
        if w == n:
            assert all(mixed_digits(rank, ext)), (rank, ext)
        R, G, touched = ref_sliced(net, legs, sl, seed)
        res, g = sp.vjp(seed, rank, w, allreduce=False)
        check("sliced gradient", res.to_numpy(), R, tau, f"{legs} slices {sl[:4]} value")
        for l in range(len(G)):
            check("sliced gradient", g[l], G[l], tau, f"{legs} slices {sl[:4]} leaf {l}")
            assert not np.any(g[l][~touched[l]]), (name, legs, rank, w, l)
    if net.flat:
        fp = SlicedPlan(net.tn, net.path, legs, ctx=c)
        R, _, _ = ref_sliced(net, legs, range(n), seed)
        check("sliced forward", fp.run().to_numpy(), R, tau, f"{legs}")
        R, _, _ = ref_sliced(net, legs, range(1, n, world), seed)
        check("sliced forward", fp.run(1, world, allreduce=False).to_numpy(), R, tau, f"{legs} rank 1 of {world}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_staging(ctxs, name):
    """set_leaves and stage_instances from torch CUDA tensors give the bits host staging gives: a plain plan (run and
    run_batch) and a gradient plan (run and vjp)"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    net = get(name)
    c = ctx_of(ctxs, net)
    dev = {l: torch.from_numpy(x).cuda() for l, x in enumerate(net.xs)}
    zeros = with_payloads(net.tn, [np.zeros_like(x) for x in net.xs])
    plain = NetworkPlan(net.tn, net.path, ctx=c)
    plain.stage(net.tn)
    want = plain.run().to_numpy()
    plain.stage(zeros)
    plain.set_leaves(dev)
    assert np.array_equal(plain.run().to_numpy(), want), name
    xss = instances(net, 3)
    plain.stage_slices([with_payloads(net.tn, xs) for xs in xss])
    want_rows = plain.run_batch(0, 3)[1].to_numpy()
    plain.stage_instances(zeros, {l: torch.from_numpy(np.stack([xs[l] for xs in xss])).cuda()
                                  for l in range(len(net.xs))}, 3)
    assert np.array_equal(plain.run_batch(0, 3)[1].to_numpy(), want_rows), name
    seed = crandn(nrng(name, 17), result_dims(net))
    grad = NetworkPlan.for_gradients(net.tn, net.path, ctx=c)
    grad.stage(net.tn)
    want = grad.run().to_numpy()
    want_g = grad.vjp(seed)
    grad.stage(zeros)
    grad.set_leaves(dev)
    assert np.array_equal(grad.run().to_numpy(), want), name
    got_g = grad.vjp(seed)
    for l in want_g:
        assert np.array_equal(got_g[l], want_g[l]), (name, l)


# ================================================================================================================
# 5. the C++ mirror's derivative methods
# ================================================================================================================
def cpp_network():
    """the network test_host_api.cpp --deriv builds, with its payload, tangent and seed formulas (exact in double)"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    spec = [([0, 1, 9], [3, 2, 2]), ([1, 2, 3], [2, 5, 1]), ([2, 4, 5], [5, 3, 2]), ([4, 0, 6, 3], [3, 3, 2, 1]),
            ([5, 7], [2, 7]), ([7, 6, 8], [7, 2, 3])]
    lv = [matrix_leaf(legs, dims, [complex(((7 * l + 3 * e) % 11 - 5) / 4, ((5 * l + 2 * e) % 13 - 6) / 8)
                                   for e in range(int(np.prod(dims)))]) for l, (legs, dims) in enumerate(spec)]
    tn = Tensor.new_composite([Tensor.new_composite(lv[0:2]), Tensor.new_composite([lv[2]]), lv[3],
                               Tensor.new_composite(lv[4:6])])
    path = ContractionPath({0: ContractionPath.simple([(0, 1)]), 1: ContractionPath.simple([]),
                            3: ContractionPath.simple([(0, 1)])}, [(0, 1), (0, 2), (0, 3)])
    net = Net("cpp_mirror", tn, path, deep=2)
    wrt = [0, 2, 5]
    tans = {l: np.array([complex(((3 * l + 5 * e) % 7 - 3) / 2, ((l + 4 * e) % 9 - 4) / 4)
                         for e in range(net.xs[l].size)]).reshape(net.xs[l].shape) for l in wrt}
    dims = result_dims(net)
    seed = np.array([complex(((2 * r) % 5 - 2) / 2, ((3 * r) % 7 - 3) / 4) for r in range(6)]).reshape(dims)
    seed_tan = np.array([complex(((r + 1) % 3 - 1) / 2, ((5 * r) % 4 - 1.5) / 2) for r in range(6)]).reshape(dims)
    return net, wrt, tans, seed, seed_tan


@pytest.mark.gpu
def test_cpp_mirror_derivative_methods(ctxs, tmp_path):
    """tnc::NetworkPlan's vjp (blocks cut at the next larger offset), jvp and hvp (cut at offset + leaf elements) give the
    Python plans' results bit for bit; those are checked against the reference here too"""
    from tnc_b200.tensornetwork import NetworkPlan
    r = subprocess.run([os.path.join(ROOT, "build", "test_host_api"), "--deriv", str(tmp_path)], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0 and "HOST_DERIV_OK" in r.stdout, r.stdout
    read = lambda f: np.fromfile(tmp_path / f, dtype=np.complex128)
    net, wrt, tans, seed, seed_tan = cpp_network()
    c = ctxs[0]
    R, G = ref_grads(net, seed)
    plan = NetworkPlan.for_gradients(net.tn, net.path, wrt, ctx=c)
    plan.stage(net.tn)
    value = plan.run().to_numpy()
    g = plan.vjp(seed)
    assert np.array_equal(read("vjp_value.bin"), value.reshape(-1))
    check("c++ mirror", value, R, TAU)
    assert sorted(g) == wrt
    for l in wrt:
        assert np.array_equal(read(f"vjp_{l}.bin"), g[l].reshape(-1)), l
        check("c++ mirror", g[l], G[l], TAU, f"G {l}")
    plan = NetworkPlan.for_tangents(net.tn, net.path, wrt, ctx=c)
    plan.stage(net.tn)
    v, t = plan.jvp(tans)
    assert np.array_equal(read("jvp_value.bin"), v.to_numpy().reshape(-1))
    assert np.array_equal(read("jvp_tangent.bin"), t.reshape(-1))
    check("c++ mirror", t, ref_jvp(net, tans)[1], TAU, "Ṙ")
    plan = NetworkPlan.for_hvp(net.tn, net.path, wrt, ctx=c)
    plan.stage(net.tn)
    value, tangent, g, dg = plan.hvp(tans, seed, seed_tan)
    assert np.array_equal(read("hvp_value.bin"), value.reshape(-1))
    assert np.array_equal(read("hvp_tangent.bin"), tangent.reshape(-1))
    _, Gd = ref_hvp(net, tans, seed, seed_tan)
    for l in wrt:
        assert np.array_equal(read(f"hvp_grad_{l}.bin"), g[l].reshape(-1)), l
        assert np.array_equal(read(f"hvp_dgrad_{l}.bin"), dg[l].reshape(-1)), l
        check("c++ mirror", dg[l], Gd[l], TAU, f"Ġ {l}")


def test_cpp_mirror_network_reference():
    """the formulas of the C++ network: a nested, mixed-extent network whose reference agrees with einsum"""
    net, wrt, tans, seed, seed_tan = cpp_network()
    assert [x.size for x in net.xs] == [12, 10, 30, 18, 14, 42]
    assert result_dims(net) in ((2, 3), (3, 2))
    assert rel_err(ref_value(net)[1], einsum_value(net)) <= 1e-13


@pytest.mark.gpu
def test_zz_report():
    """runs last: prints the worst error each plan kind reached over the corpus and the engine counts of the counted
    calls (the pair-by-pair forward passes and the every-leaf backward passes)"""
    for kind, e in sorted(WORST.items()):
        print(f"worst error {kind}: {e:.3g}")
    print("engine counts:", ENGINES)
