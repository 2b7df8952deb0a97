"""Repeatability harness for the GPU tests: what a library call read and wrote, and memory poisoning.

  digest        position- and bit-sensitive int64 digest of a tensor, computed on the device
  Tracer        wraps ops._call and ops._p; per library call: name, scalar arguments and, per tensor argument, shape,
                dtype and digests before and after the call.  mode="check" also reruns every call from its restored
                pre-state over re-poisoned pool memory and reports the arguments that came out different
  poison_pool   fills the memory the stream-ordered pool keeps (og_work_alloc's workspaces) with a byte pattern
  poisoned      context: torch.empty / empty_like / Tensor.new_empty / ops._empty_slack return pattern-filled memory
  diagnose      the earliest call of two traced runs whose read-only inputs agree but whose output differs where a
                later call reads it

Run as a script (``python repeat.py OUT.json BATCH``) it is the child of test_step_a_bitwise_across_processes.
"""
import contextlib
import ctypes
import sys
import weakref
from collections import namedtuple

import torch

# ---------------------------------------------------------------------------------------------------------------------
# digests
# ---------------------------------------------------------------------------------------------------------------------
_K = -7046029254386353131           # 0x9E3779B97F4A7C15 as int64 (odd)


def digest(t):
    """int64 device scalar: sum_i w_i * (2i + 1) * K over the 32-bit words w_i (taken unsigned) of t's bytes in memory
    order (zero-padded to a whole word), wrapping modulo 2^64.  Every multiplier is odd, hence invertible modulo 2^64:
    a change of any one word, i.e. of any bit, changes the digest, and so does a move of a word to another index."""
    b = t.detach().contiguous().reshape(-1).view(torch.uint8)
    if b.numel() % 4:
        b = torch.cat((b, b.new_zeros(4 - b.numel() % 4)))
    w = b.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    m = (torch.arange(w.numel(), device=w.device, dtype=torch.int64) * 2 + 1) * _K
    return (w * m).sum()


_INT_OF_SIZE = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits(t):
    """t's elements as integers of the same width (flat): equal bits compare equal, NaN and -0.0 included."""
    return t.detach().contiguous().reshape(-1).view(_INT_OF_SIZE[t.element_size()])


# ---------------------------------------------------------------------------------------------------------------------
# the stream-ordered pool (the driver API through ctypes: torch exposes no handle to cudaMallocAsync's default pool)
# ---------------------------------------------------------------------------------------------------------------------
_POOL_RELEASE_THRESHOLD, _POOL_RESERVED_CURRENT, _POOL_USED_CURRENT = 4, 5, 7
_POINTER_MEMORY_TYPE = 2
_cu = None


def _driver():
    global _cu
    if _cu is None:
        _cu = ctypes.CDLL("libcuda.so.1")
        for name in ("cuMemAllocAsync", "cuMemFreeAsync", "cuMemsetD8Async", "cuStreamSynchronize",
                     "cuDeviceGetDefaultMemPool", "cuMemPoolGetAttribute", "cuMemPoolSetAttribute", "cuCtxGetDevice",
                     "cuPointerGetAttribute", "cuMemcpyDtoDAsync_v2"):
            getattr(_cu, name).restype = ctypes.c_int
    return _cu


def _ok(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed with CUresult %d" % (what, rc))


def _pool():
    cu = _driver()
    torch.cuda.init()
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    _ok(cu.cuCtxGetDevice(ctypes.byref(dev)), "cuCtxGetDevice")
    _ok(cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev), "cuDeviceGetDefaultMemPool")
    return pool


def _pool_attr(pool, attr):
    v = ctypes.c_uint64()
    _ok(_driver().cuMemPoolGetAttribute(pool, attr, ctypes.byref(v)), "cuMemPoolGetAttribute")
    return v.value


def poison_pool(pattern, big=256 << 20):
    """Fill what the device's default pool holds with ``pattern`` bytes: one ``big`` block, then blocks of the largest
    power of two that fits the rest of what the pool holds, until (nearly) all of it is handed out; all are filled,
    freed on the current stream and synchronised.  The next og_work_alloc calls are then carved out of poisoned
    memory.  A block the pool's free pieces cannot hold makes it reserve more; the block size is then halved, and
    the fill ends when a 4 KiB block does not fit (smaller pieces stay unpoisoned).  The pool is first told to keep
    what is freed (the release threshold og_work_alloc sets on the same, per-process pool), or the freed blocks
    would go back to the driver at the synchronisation."""
    cu, pool = _driver(), _pool()
    keep = ctypes.c_uint64(2 ** 64 - 1)
    _ok(cu.cuMemPoolSetAttribute(pool, _POOL_RELEASE_THRESHOLD, ctypes.byref(keep)), "cuMemPoolSetAttribute")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda.current_stream().synchronize()
    blocks, size, cap = [], big, big
    for _ in range(2048):
        r0 = _pool_attr(pool, _POOL_RESERVED_CURRENT)
        if blocks:
            gap = r0 - _pool_attr(pool, _POOL_USED_CURRENT)
            if gap < 4096:
                break
            size = min(cap, 1 << (gap.bit_length() - 1))
        p = ctypes.c_uint64()
        _ok(cu.cuMemAllocAsync(ctypes.byref(p), ctypes.c_size_t(size), stream), "cuMemAllocAsync")
        blocks.append((p, size))
        if blocks[1:] and _pool_attr(pool, _POOL_RESERVED_CURRENT) > r0:
            if size <= 4096:
                break
            cap = size // 2
    for p, size in blocks:
        _ok(cu.cuMemsetD8Async(p, ctypes.c_ubyte(pattern), ctypes.c_size_t(size), stream), "cuMemsetD8Async")
    for p, _ in blocks:
        _ok(cu.cuMemFreeAsync(p, stream), "cuMemFreeAsync")
    _ok(cu.cuStreamSynchronize(stream), "cuStreamSynchronize")


def read_unwritten_pool_bytes(out):
    """A fabricated library call for the mutant test: copies ``out.nbytes`` bytes of a fresh, unwritten pool block
    into ``out`` (in bounds on both sides; only the values it reads are undefined)."""
    cu = _driver()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n = out.numel() * out.element_size()
    p = ctypes.c_uint64()
    _ok(cu.cuMemAllocAsync(ctypes.byref(p), ctypes.c_size_t(n), stream), "cuMemAllocAsync")
    _ok(cu.cuMemcpyDtoDAsync_v2(ctypes.c_uint64(out.data_ptr()), p, ctypes.c_size_t(n), stream), "cuMemcpyDtoDAsync")
    _ok(cu.cuMemFreeAsync(p, stream), "cuMemFreeAsync")


def is_device_pointer(ptr):
    t = ctypes.c_uint()
    return _driver().cuPointerGetAttribute(ctypes.byref(t), _POINTER_MEMORY_TYPE, ctypes.c_uint64(ptr)) == 0


# ---------------------------------------------------------------------------------------------------------------------
# Python-side allocations
# ---------------------------------------------------------------------------------------------------------------------
def fill_bytes(t, pattern):
    if t.numel():
        t.detach().reshape(-1).view(torch.uint8).fill_(pattern)
    return t


@contextlib.contextmanager
def poisoned(pattern):
    """torch.empty, torch.empty_like, Tensor.new_empty and ops._empty_slack (its 512-byte slack included) return
    memory filled with ``pattern`` bytes while the context is active."""
    from objgan_b200 import ops
    real = torch.empty, torch.empty_like, torch.Tensor.new_empty, ops._empty_slack

    def empty(*a, **k):
        return fill_bytes(real[0](*a, **k), pattern)

    def empty_like(*a, **k):
        return fill_bytes(real[1](*a, **k), pattern)

    def new_empty(self, *a, **k):
        return fill_bytes(real[2](self, *a, **k), pattern)

    def empty_slack(shape, device):
        t = real[3](shape, device)
        fill_bytes(t._base if t._base is not None else t, pattern)
        return t
    torch.empty, torch.empty_like, torch.Tensor.new_empty, ops._empty_slack = empty, empty_like, new_empty, empty_slack
    try:
        yield
    finally:
        torch.empty, torch.empty_like, torch.Tensor.new_empty, ops._empty_slack = real


# ---------------------------------------------------------------------------------------------------------------------
# the call tracer
# ---------------------------------------------------------------------------------------------------------------------
# One library call.  args: per tensor argument (position, shape, dtype); pre / post: their digests (ints) before and
# after the call; keys: a per-run identity of each argument's memory (data pointer, shape, dtype)
Call = namedtuple("Call", "name scalars args keys pre post")
# A call whose rerun over re-poisoned memory wrote different values: per differing argument (position, shape, dtype,
# differing elements, first differing flat index, largest |difference| relative to max |first run|)
Mismatch = namedtuple("Mismatch", "index name args diffs")
# pointer tables: entry -> (argument holding the int64 table, row width, columns that hold device pointers)
TABLES = {"og_amax_multi": (0, 4, (0, 2)), "og_pack_weights_f16_multi": (0, 14, (0, 1, 2, 3))}


class Tracer:
    """Records every library call issued inside ``with Tracer(...)``.

    Each call learns which tensors are behind its pointer arguments: ops._p registers the tensor it is asked for
    (held until the call), torch.empty registers what it returns (weakly: raw offsets into such a tensor, like
    EncConv.folded's og_bn_fold destinations, map to it), PackPlan.run registers its jobs' tensors, and the pointer
    tables of TABLES are read back and mapped like arguments.  A device pointer that maps to no tensor is a gap of
    the tracer and is listed in ``unmapped``; host pointers (ctypes arrays of tap tables) are skipped.

    mode "digest": digests are taken on the stream of the call, so branches on other streams keep running
    concurrently; ``calls`` holds the Call records (digests resolved at exit).
    mode "check": before each call the tracer synchronises, clones the arguments, poisons the pool with
    patterns[0] and runs the call; it clones the results, restores the pre-state, poisons the pool with patterns[1]
    and runs the call again.  Every argument must come out bitwise equal to the first run, or, for the entries of
    ``tolerant`` (name -> relative tolerance), within that fraction of the largest magnitude.  ``mismatches`` lists
    every call that failed."""

    def __init__(self, mode="digest", patterns=(0xFF, 0x5A), tolerant=None):
        assert mode in ("digest", "check")
        self.mode, self.patterns, self.tolerant = mode, patterns, dict(tolerant or {})
        self.calls, self.mismatches, self.unmapped = [], [], []
        self._held, self._weak, self._pending = [], {}, []

    # -- tensor registry -------------------------------------------------------------------------------------------
    def register(self, t, hold=True):
        if t is None or not torch.is_tensor(t) or not t.is_cuda:
            return
        if hold:
            self._held.append(t)
        ptr = t.data_ptr()
        self._weak.pop(ptr, None)
        self._weak[ptr] = weakref.ref(t)

    def _live(self):
        for t in reversed(self._held):
            yield t
        for r in reversed(list(self._weak.values())):
            t = r()
            if t is not None:
                yield t

    def lookup(self, ptr):
        """The tensor behind a device pointer: the latest registered tensor starting there, else the latest whose
        storage contains it."""
        for t in self._live():
            if t.data_ptr() == ptr:
                return t
        for t in self._live():
            st = t.untyped_storage()
            if st.data_ptr() <= ptr < st.data_ptr() + st.nbytes():
                return t
        return None

    def _prune(self):
        self._weak = {p: r for p, r in self._weak.items() if r() is not None}

    # -- the wrapped entry points ----------------------------------------------------------------------------------
    def __enter__(self):
        from objgan_b200 import lib, ops
        self._ops, self._lib = ops, lib
        self._real = ops._call, ops._p, torch.empty, ops.PackPlan.run
        real_call, real_p, real_empty, real_run = self._real

        def p(t):
            self.register(t)
            return real_p(t)

        def empty(*a, **k):
            t = real_empty(*a, **k)
            self.register(t, hold=False)
            return t

        def run(plan):
            for j in plan.jobs:
                for t in (j.w, j.hi, j.lo, j.amax):
                    self.register(t)
            return real_run(plan)

        def call(name, *args):
            try:
                return self._traced(real_call, name, args)
            finally:
                self._held = []
        ops._call, ops._p, torch.empty, ops.PackPlan.run = call, p, empty, run
        return self

    def __exit__(self, *exc):
        self._ops._call, self._ops._p, torch.empty, self._ops.PackPlan.run = self._real
        if self._pending:
            torch.cuda.synchronize()        # the digests of calls on branch streams
            ds = [d for c in self._pending for d in c.pre + c.post]
            flat = torch.stack(ds).tolist() if ds else []
            i = 0
            for c in self._pending:
                n = len(c.pre)
                self.calls.append(c._replace(pre=flat[i:i + n], post=flat[i + n:i + 2 * n]))
                i += 2 * n
            self._pending = []
        return False

    def tensors_of(self, name, args):
        """[(position, tensor)] of the distinct tensors behind a call's pointer arguments; a table's pointers get the
        position (table argument, row, column)."""
        types = self._lib.get().protos[name][:-1]
        ptrs = [(i, a) for i, (a, ty) in enumerate(zip(args, types)) if ty is ctypes.c_void_p and a]
        if name in TABLES:
            arg, width, cols = TABLES[name]
            rows = self.lookup(args[arg]).view(-1, width).tolist()
            ptrs += [((arg, r, c), row[c]) for r, row in enumerate(rows) for c in cols]
        out, seen = [], set()
        for pos, ptr in ptrs:
            t = self.lookup(ptr)
            if t is None:
                if is_device_pointer(ptr):
                    self.unmapped.append((name, pos))
                continue
            key = (t.data_ptr(), tuple(t.shape), t.dtype)
            if key not in seen:
                seen.add(key)
                out.append((pos, t))
        return out

    def _traced(self, real, name, args):
        if len(self._weak) > 4096:
            self._prune()
        ts = self.tensors_of(name, args)
        scalars = tuple(a for a, ty in zip(args, self._lib.get().protos[name]) if ty is not ctypes.c_void_p)
        desc = [(pos, tuple(t.shape), str(t.dtype).replace("torch.", "")) for pos, t in ts]
        keys = [(t.data_ptr(), tuple(t.shape), t.dtype) for _, t in ts]
        if self.mode == "digest":
            pre = [digest(t) for _, t in ts]
            real(name, *args)
            post = [digest(t) for _, t in ts]
            self._pending.append(Call(name, scalars, desc, keys, pre, post))
            return
        torch.cuda.synchronize()
        before = [t.clone() for _, t in ts]
        poison_pool(self.patterns[0])
        real(name, *args)
        torch.cuda.synchronize()
        first = [t.clone() for _, t in ts]
        for (_, t), b in zip(ts, before):
            t.data.copy_(b)         # through .data: autograd's version counter of t stays as the first run left it
        poison_pool(self.patterns[1])
        real(name, *args)
        torch.cuda.synchronize()
        diffs = []
        tol = self.tolerant.get(name)
        for (pos, t), f, d in zip(ts, first, desc):
            ne = bits(t) != bits(f)
            n = int(ne.sum())
            if not n:
                continue
            rel = None
            if t.is_floating_point():
                a, b = t.double().reshape(-1), f.double().reshape(-1)
                rel = float((a - b).abs().nan_to_num(float("inf")).max() / b.abs().nan_to_num(0).max().clamp(min=1e-30))
                if tol is not None and rel <= tol:
                    continue
            diffs.append((pos, d[1], d[2], n, int(ne.nonzero()[0, 0]), rel))
        if diffs:
            self.mismatches.append(Mismatch(len(self.calls), name, desc, diffs))
        self.calls.append(Call(name, scalars, desc, keys, [], []))


def report(mismatches):
    return "\n".join("call %d %s args %s: %s" % (m.index, m.name, [d[1:] for d in m.args],
                                                 "; ".join("arg %s %s %s: %d elements differ, first at %s, max rel %s"
                                                           % d for d in m.diffs)) for m in mismatches)


def _span(key):
    ptr, shape, dtype = key
    n = 1
    for d in shape:
        n *= d
    return ptr, ptr + n * torch.empty((), dtype=dtype).element_size()


def diagnose(a, b):
    """Compare two Tracer("digest") call lists of the same work.  Returns (index, text) of the earliest call whose
    read-only arguments (pre digest = post digest in both runs) agree between the runs while a tensor it wrote
    differs, and differs again when a later call reads it (as a read-only argument over the same memory), or
    (None, text) when there is no such call.  A written tensor that differs only until a later call completes it
    (outputs written in parts) is not a culprit."""
    def ro(x, y, k):
        return x.pre[k] == x.post[k] and y.pre[k] == y.post[k]

    def later_read(i, key):
        """(index, name) of the first later read-only use of key's memory that differs between the runs, or None when
        a later use covering all of it agrees first."""
        lo, hi = _span(key)
        for j in range(i + 1, len(a)):
            for kk, key2 in enumerate(a[j].keys):
                lo2, hi2 = _span(key2)
                if lo2 >= hi or lo >= hi2:
                    continue
                covers = lo2 <= lo and hi <= hi2
                if ro(a[j], b[j], kk):
                    if a[j].pre[kk] != b[j].pre[kk]:
                        return j, a[j].name
                    if covers:
                        return None
                elif covers and a[j].post[kk] == b[j].post[kk]:
                    return None
        return None

    for i, (x, y) in enumerate(zip(a, b)):
        if (x.name, x.scalars, x.args) != (y.name, y.scalars, y.args):
            return None, "the call sequences part at call %d: %s%s vs %s%s" % (i, x.name, x.args, y.name, y.args)
        if any(x.pre[k] != y.pre[k] for k in range(len(x.args)) if ro(x, y, k)):
            continue
        for k in range(len(x.args)):
            if ro(x, y, k) or x.post[k] == y.post[k]:
                continue
            read = later_read(i, x.keys[k])
            if read is not None:
                return i, ("call %d %s (scalars %s) read agreeing inputs and wrote a differing %s; call %d %s reads it"
                           % (i, x.name, x.scalars, x.args[k], read[0], read[1]))
    if len(a) != len(b):
        return None, "the runs issued %d and %d calls" % (len(a), len(b))
    return None, "no call of the traced runs read agreeing inputs and wrote a differing tensor that is read later"


# ---------------------------------------------------------------------------------------------------------------------
# Step-A runs
# ---------------------------------------------------------------------------------------------------------------------
SEED = 1234


def step_a_setup(batch, seed=SEED):
    """A seeded StepATrainer and its device batch, built like bench.py's: compact host batch, heat maps rebuilt on the
    device, CA_NET noise drawn on the device."""
    from objgan_b200 import synth, trainer
    t = trainer.StepATrainer(device="cuda", seed=seed)
    full = synth.make_inputs(batch, seed=seed, parity=False)
    full.pop("eps")
    return t, trainer.pin(synth.compact(full))


def step_a_state(t, out):
    """name -> tensor: the losses, fake images, bG flat/grad/m/v/avg, every bD flat/m/v and every BatchNorm buffer."""
    s = {k: out[k] for k in ("errPatD0", "errPatD1", "errPatD2", "errG", "kl")}
    s.update({"fake_imgs%d" % i: f for i, f in enumerate(out["fake_imgs"])})
    for n in ("flat", "grad", "m", "v", "avg"):
        s["bG." + n] = getattr(t.bG, n)
    for i, b in enumerate(t.bD):
        for n in ("flat", "m", "v"):
            s["bD%d.%s" % (i, n)] = getattr(b, n)
    for j, net in enumerate([t.netG, *t.netsPatD]):
        for n, buf in net.named_buffers():
            s["net%d.%s" % (j, n)] = buf
    return {k: v.detach().clone() for k, v in s.items()}


def _child(path, batch):
    """Two eager Step-A steps of one trainer, and a capture and two replays of a second one from the same seed (a
    trainer captures before its first eager step: autograd's AccumulateGrad nodes keep the stream of their first
    backward); writes the state digests after each step."""
    import json
    res = {}
    t, host = step_a_setup(batch)
    dev = t.to_device(host)
    for i in range(2):
        res["eager%d" % i] = {k: int(digest(v)) for k, v in step_a_state(t, t.step(dev)).items()}
    del t, dev
    t, host = step_a_setup(batch)
    dev = t.to_device(host)
    t.capture(dev)
    for i in range(2):
        res["replay%d" % i] = {k: int(digest(v)) for k, v in step_a_state(t, t.step(dev)).items()}
    torch.cuda.synchronize()
    with open(path, "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    import os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    _child(sys.argv[1], int(sys.argv[2]))
