"""Every public entry point off the default stream, and the model's cached device state handed across streams.

The library launches on the caller's current stream, and the model keeps device state between calls (packed weights,
attention constants, coordinate tables, NIQE tables, captured graphs) that one stream makes and others read.  Each race
here puts a bounded torch.cuda._sleep on one stream so that work queued behind it is still pending while the host
enqueues the rest: a launch on the wrong stream, or a read that is not ordered after the write it needs, then sees
memory that is not written yet.  The reference of every comparison is the same call on the default stream, and every
comparison is bit for bit.  A race is only conclusive when the delay is still running after the host has enqueued all
the work under test; the tests check that once and never retry.

Part A: each public entry point on a side stream S, its inputs made on S behind the delay; every stream argument the
  library receives is S (a recorder stands in for capi.lib()).  Mutation control: grl_tc_attn routed to another stream
  must change the output.
Part B: an entry produced behind a delay on stream A and used by a forward on stream B (read before written).
Part C: an entry used behind a delay, then dropped and its memory reallocated on the default stream (reuse after free).
Part D: two streams replaying one captured graph at once.
Coverage guard: every CUDA tensor the model or the package's module-level caches keep between calls is held under the
  ordering mechanism (streams.Produced).
"""
import copy
import ctypes
import os
import re
import sys

import pytest
import torch

from support import build

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NIQE_PARAMS = os.path.join(GOLD, "niqe_pris_params.npz")
DELAY_S, MAX_DELAY_S = 0.2, 0.25
INCONCLUSIVE = "inconclusive: delay ended before the consumer was enqueued"
R1, R2, R3 = (32, 32), (32, 48), (48, 48)  # padded sizes: R1 the model's img_size (its table buffers), R2 / R3 cached


class Env:
    """The session's streams and the delay calibrated once with CUDA events."""

    def __init__(self):
        self.S, self.A, self.B, self.other = (torch.cuda.Stream() for _ in range(4))
        torch.cuda._sleep(1000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        probe = 1 << 22
        e0.record()
        torch.cuda._sleep(probe)
        e1.record()
        e1.synchronize()
        self.cycles_per_ms = probe / e0.elapsed_time(e1)
        self.cycles = int(min(DELAY_S, MAX_DELAY_S) * 1e3 * self.cycles_per_ms)

    def delay(self, stream, ms=None):
        """A bounded sleep on `stream` (DELAY_S, or `ms`); returns the event recorded right after it."""
        cycles = self.cycles if ms is None else min(self.cycles, int(ms * self.cycles_per_ms))
        ev = torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            torch.cuda._sleep(cycles)
            ev.record(stream)
        return ev


@pytest.fixture(scope="module")
def env(pkg, device):
    from grl_image_restoration_b200 import capi

    if capi.lib().grl_device_ok() != 1:
        pytest.skip("the tensor-core path needs sm_90")
    return Env()


def streamed_entry_points():
    """The C entry points whose last parameter is the stream (include/grl_b200.h)."""
    from grl_image_restoration_b200 import capi

    with open(capi.HEADER_PATH) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return {m.group(1) for m in re.finditer(r"\b(grl_[a-z0-9_]+)\s*\(([^)]*)\)", src) if m.group(2).rstrip().endswith("stream")}


class StreamRecorder:
    """Stands in for capi.lib(): records the stream argument of every launching entry point and forwards the call;
    `reroute` = (name, stream handle) launches that entry point on another stream (the mutation control)."""

    def __init__(self, lib, streamed, reroute=None):
        self._lib, self._streamed, self._reroute, self.calls = lib, streamed, reroute, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in self._streamed:
            return fn

        def call(*args):
            s = args[-1]
            self.calls.append((name, s.value if isinstance(s, ctypes.c_void_p) else s))
            if self._reroute and name == self._reroute[0]:
                args = args[:-1] + (ctypes.c_void_p(self._reroute[1]),)
            return fn(*args)

        return call


def clone(v):
    if isinstance(v, torch.Tensor):
        return v.clone()
    if isinstance(v, (list, tuple)):
        return type(v)(clone(e) for e in v)
    return v


def same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    return a == b


def on_side(env, monkeypatch, fn, srcs, reroute=None):
    """fn(*inputs) under `with torch.cuda.stream(env.S)` behind a delay, the inputs copied from the default-stream
    sources `srcs` on S after the delay.  Returns (output, recorded calls); fails when the race was not conclusive."""
    from grl_image_restoration_b200 import capi

    torch.cuda.synchronize()
    rec = StreamRecorder(capi.lib(), streamed_entry_points(),
                         None if reroute is None else (reroute, env.other.cuda_stream))
    with monkeypatch.context() as mp:
        mp.setattr(capi, "lib", lambda: rec)
        ev = env.delay(env.S)
        with torch.cuda.stream(env.S):
            out = fn(*clone(srcs))
        pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, INCONCLUSIVE
    return out, rec.calls


def side_stream_case(env, monkeypatch, fn, make, graph_only=False):
    """Part A for one entry point: the default-stream result of make(seed) inputs, a warm-up on S with other inputs
    (so that memory S reuses holds other values), then the race.  Every launch must be on S."""
    srcs = make(1)
    ref = fn(*srcs)
    torch.cuda.synchronize()
    env.S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(env.S):
        fn(*make(2))
    out, calls = on_side(env, monkeypatch, fn, srcs)
    wrong = [(n, s) for n, s in calls if s != env.S.cuda_stream]
    assert not wrong, f"launched off the current stream: {wrong[:5]}"
    assert graph_only or calls, "no library launch recorded"
    assert same(out, ref), "differs from the default-stream result"


# ---------------------------------------------------------------------------------------------------------- models


def micro_model(pkg, oracle, precision, **kw):
    m = build(pkg, oracle, pkg.configs.micro_config(), "cuda", precision, style="init", **kw)
    m.use_cuda_graph = False
    return m


def rand(seed, *shape, u8=False):
    g = torch.Generator().manual_seed(seed)
    if u8:
        return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).cuda()
    return torch.rand(*shape, generator=g).cuda()


MODEL_CASES = [(p, f, e, g) for p in ("fp32", "fp16", "bf16") for f in ("rgb", "rggb") for e in (False, True)
               for g in ((False,) if p == "fp32" else (False, True))]


@pytest.mark.parametrize("precision,fmt,ensemble,graph", MODEL_CASES)
def test_model_on_side_stream(pkg, oracle, env, monkeypatch, precision, fmt, ensemble, graph):
    m = micro_model(pkg, oracle, precision, input_format=fmt, self_ensemble=ensemble)
    m.use_cuda_graph = graph
    shape = (2, 4, 12, 20) if fmt == "rggb" else (2, 3, 24, 40)
    side_stream_case(env, monkeypatch, m, lambda s: (rand(s, *shape),), graph_only=graph and not ensemble)


def _entry_cases(pkg, oracle):
    from grl_image_restoration_b200 import functional as K, metrics, tiling

    m = micro_model(pkg, oracle, "fp16")
    sizes = [(24, 40), (17, 30), (24, 40), (9, 13)]
    flist = lambda s: ([rand(s + i, 3, h, w) for i, (h, w) in enumerate(sizes)],)  # noqa: E731
    ulist = lambda s: ([rand(s + i, h, w, 3, u8=True) for i, (h, w) in enumerate(sizes)],)  # noqa: E731
    pair = lambda s: (rand(s, 2, 3, 40, 48), rand(s + 9, 2, 3, 40, 48))  # noqa: E731
    return {
        "forward_u8": (m.forward_u8, lambda s: (rand(s, 2, 24, 40, 3, u8=True),)),
        "forward_list": (m.forward_list, flist),
        "forward_list_u8": (m.forward_list_u8, ulist),
        "forward_tile": (lambda x: tiling.forward_tile(m, x, 32, 8), lambda s: (rand(s, 1, 3, 40, 56),)),
        "forward_tile_u8": (lambda x: tiling.forward_tile_u8(m, x, 32, 8), lambda s: (rand(s, 1, 40, 56, 3, u8=True),)),
        "forward_tile_list": (lambda xs: tiling.forward_tile_list(m, xs, 16, 4), flist),
        "forward_tile_list_u8": (lambda xs: tiling.forward_tile_list_u8(m, xs, 16, 4), ulist),
        "jpeg_roundtrip": (lambda x: K.jpeg_roundtrip(x, 30), lambda s: (rand(s, 2, 24, 40, 3, u8=True),)),
        "jpeg_roundtrip_list": (lambda xs: K.jpeg_roundtrip_list(xs, 30), ulist),
        "demosaic": (K.demosaic, lambda s: (rand(s, 2, 4, 12, 20),)),
        "psnr_fused": (lambda a, b: metrics.psnr_fused(a, b, 2), pair),
        "psnrb_fused": (metrics.psnrb_fused, pair),
        "ssim_fused": (lambda a, b: metrics.ssim_fused(a, b, 2), pair),
        "niqe_features": (lambda x: metrics.niqe_features(x, NIQE_PARAMS, 0), lambda s: (rand(s, 2, 3, 96, 192),)),
        "validation_metrics_fused": (lambda a, b: metrics.validation_metrics_fused(a, b, 2, True), pair),
    }


ENTRIES = ["forward_u8", "forward_list", "forward_list_u8", "forward_tile", "forward_tile_u8", "forward_tile_list",
           "forward_tile_list_u8", "jpeg_roundtrip", "jpeg_roundtrip_list", "demosaic", "psnr_fused", "psnrb_fused",
           "ssim_fused", "niqe_features", "validation_metrics_fused"]


@pytest.mark.parametrize("entry", ENTRIES)
def test_entry_point_on_side_stream(pkg, oracle, env, monkeypatch, entry):
    fn, make = _entry_cases(pkg, oracle)[entry]
    side_stream_case(env, monkeypatch, fn, make)


def test_misstreamed_launch_is_caught(pkg, oracle, env, monkeypatch):
    """Mutation control: the same race with every grl_tc_attn launch put on another stream must not match."""
    m = micro_model(pkg, oracle, "fp16")
    srcs = (rand(1, 2, 3, 24, 40),)
    ref = m(*srcs)
    torch.cuda.synchronize()
    env.S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(env.S):
        m(rand(2, 2, 3, 24, 40))
    out, calls = on_side(env, monkeypatch, m, srcs, reroute="grl_tc_attn")
    assert any(n == "grl_tc_attn" for n, _ in calls)
    assert not same(out, ref), "a launch on the wrong stream went unnoticed: the delay does not expose it"


# ---------------------------------------------------------------------------------------------------------- Part B


def x_at(seed, size, batch=1):
    return rand(seed, batch, 3, *size)


def handoff(env, model, xa, xb, call=None):
    """Producer call on A behind a delay, then the consumer call on B, with no host synchronisation between them."""
    call = call or model
    torch.cuda.synchronize()
    ev = env.delay(env.A)
    with torch.cuda.stream(env.A):
        ya = call(xa)
    with torch.cuda.stream(env.B):
        yb = call(xb)
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, INCONCLUSIVE
    return ya, yb


def warm_streams(env, model, x):
    """One call on each of A and B, so that their memory pools hold blocks with other values."""
    for s in (env.A, env.B):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model(x)
    torch.cuda.synchronize()


HANDOFF = [("constants", "fp16"), ("constants", "bf16"), ("set_precision", "fp16"), ("set_precision", "bf16"),
           ("edit", "fp16"), ("edit", "bf16"), ("edit", "fp32"), ("new_resolution", "fp16"),
           ("new_resolution", "bf16"), ("new_resolution", "fp32")]


@pytest.mark.parametrize("case,precision", HANDOFF)
def test_cross_stream_handoff(pkg, oracle, env, case, precision):
    """Hazard 1: a cache entry the producer on A rebuilds behind the delay is read by the consumer on B; both outputs
    equal the default-stream reference.  constants: R1 and R2 warmed, the forward at R1 rebuilds the attention constants;
    set_precision / edit: the packed weights (fp32: the im2col conv weights) are rebuilt; new_resolution: the coordinate
    tables, constants and plans of a resolution first seen on A."""
    m = micro_model(pkg, oracle, {"set_precision": "bf16" if precision == "fp16" else "fp16"}.get(case, precision))
    size = R3 if case == "new_resolution" else R1
    xa, xb = x_at(11, size), x_at(12, size)
    warm_streams(env, m, x_at(3, R2))
    if case == "constants":
        ref = (m(xa), m(xb))
        m(x_at(4, R2))
    elif case == "set_precision":
        m(x_at(4, R1))
        m.set_precision(precision)
    elif case == "edit":
        m(x_at(4, R1))
        blk = m.layers[0].blocks[1]
        with torch.no_grad():
            blk.mlp.fc1.weight.mul_(1.1)
            m.conv_first.weight.mul_(0.9)
            blk.conv.cab[0].weight.mul_(1.05)
    if case != "constants":
        torch.cuda.synchronize()
        r = copy.deepcopy(m)
        ref = (r(xa), r(xb))
        del r
    ya, yb = handoff(env, m, xa, xb)
    assert same(ya, ref[0]), "the producer's output differs from the default-stream reference"
    assert same(yb, ref[1]), "the consumer read a cache entry before its producer wrote it"


def test_niqe_tables_handoff(pkg, env):
    from grl_image_restoration_b200 import metrics

    xa, xb = rand(21, 1, 3, 96, 192), rand(22, 1, 3, 96, 192)
    f = lambda x: metrics.niqe_features(x, NIQE_PARAMS, 0)  # noqa: E731
    ref = (f(xa), f(xb))
    warm_streams(env, f, rand(23, 1, 3, 96, 96))
    metrics._niqe_cache.clear()
    ya, yb = handoff(env, None, xa, xb, call=f)
    assert same(ya, ref[0]) and same(yb, ref[1]), "NIQE features read the tables before they were uploaded"


# ---------------------------------------------------------------------------------------------------------- Part C


REUSE = [("resolution", "fp16"), ("set_precision", "fp16"), ("set_precision", "bf16"), ("edit", "fp16"),
         ("edit", "fp32"), ("eviction", "fp16"), ("eviction", "fp32")]


@pytest.mark.parametrize("case,precision", REUSE)
def test_reuse_after_free(pkg, oracle, env, case, precision):
    """Hazard 2: a forward queued on the delayed stream S reads entries made on the default stream; the default stream
    then drops them and runs a forward that allocates and writes there.  S's output must still equal the reference."""
    m = micro_model(pkg, oracle, precision)
    size = R3 if case == "eviction" else R1
    x = x_at(31, size)
    ref = m(x)
    warm_streams(env, m, x_at(3, R2))
    m(x_at(32, size))  # every entry S reads is made on the default stream
    if case == "eviction":
        m(x_at(33, R1))  # the constants are R1's: S recomputes them from R3's tables
        torch.cuda.synchronize()
        assert len(m._table_cache) < 16
    torch.cuda.synchronize()
    env.S.wait_stream(torch.cuda.current_stream())
    ev = env.delay(env.S)
    with torch.cuda.stream(env.S):
        y = m(x)
    if case == "resolution":
        m(x_at(34, R2))
    elif case == "set_precision":
        m.set_precision("bf16" if precision == "fp16" else "fp16")
        m(x_at(34, R1))
    elif case == "edit":  # weights every path reads only through its packed copy, so S's forward reads none of them
        with torch.no_grad():
            m.layers[0].blocks[1].conv.cab[0].weight.mul_(1.1)
            m.layers[0].conv.weight.mul_(0.9)
        m(x_at(34, R1))
    else:
        n = 0
        while len(m._table_cache) and (R3, "cuda:0") in {(k[0], k[1]) for k in m._table_cache}:
            m.get_table_index_mask(torch.device("cuda:0"), (16 * (4 + n), 16))
            n += 1
        m(x_at(34, (16 * (4 + n), 16)))
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, INCONCLUSIVE
    assert same(y, ref), "the delayed forward read memory that was freed and reused"


# ---------------------------------------------------------------------------------------------------------- Part D


def test_concurrent_graph_replays(pkg, oracle, env):
    """Hazard 3: one captured graph replayed from two streams at once (A delayed by about half a replay); the two
    executions would overlap without ordering, and both outputs equal the eager results."""
    m = micro_model(pkg, oracle, "fp16")
    xa, xb = rand(41, 32, 3, 192, 192), rand(42, 32, 3, 192, 192)
    ref = (m(xa), m(xb))
    m.use_cuda_graph = True
    m(xa)
    for s in (env.A, env.B):  # first replays on each stream, outside the race
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(xb)
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    m(xa)
    e1.record()
    torch.cuda.synchronize()
    d = e0.elapsed_time(e1)
    for s in (env.A, env.B):
        s.wait_stream(torch.cuda.current_stream())
    ev = env.delay(env.A, d / 2)
    with torch.cuda.stream(env.A):
        ya = m(xa)
    start_b = torch.cuda.Event(enable_timing=True)
    start_b.record(env.B)
    with torch.cuda.stream(env.B):
        yb = m(xb)
    pending = not ev.query()
    torch.cuda.synchronize()
    gap = start_b.elapsed_time(ev)  # from B's call becoming ready to A's replay starting
    print(f"\nreplay {d:.3f} ms; A's replay started {gap:.3f} ms after B's call was ready")
    assert pending and 0 < gap < d, INCONCLUSIVE + f" (or the calls would not overlap: gap {gap:.3f} ms, replay {d:.3f} ms)"
    assert same(ya, ref[0]) and same(yb, ref[1]), "concurrent replays of one graph corrupted each other"


# ---------------------------------------------------------------------------------------------------------- coverage


def unordered_tensors(root, pkg_name):
    """CUDA tensors reachable from `root` (tuples, lists, dicts, objects of the package's own classes) that are not
    among the tensors of a streams.Produced reachable the same way.  Returns (unordered paths, number ordered)."""
    from grl_image_restoration_b200.streams import Produced, tensors

    held, loose, seen = set(), [], set()

    def walk(v, path):
        if id(v) in seen:
            return
        seen.add(id(v))
        if isinstance(v, Produced):
            held.update(t.untyped_storage().data_ptr() for t in tensors(v.value) if t.is_cuda)
        elif isinstance(v, torch.Tensor):
            if v.is_cuda:
                loose.append((path, v))
        elif isinstance(v, (tuple, list)):
            for i, e in enumerate(v):
                walk(e, f"{path}[{i}]")
        elif isinstance(v, dict):
            for k, e in v.items():
                walk(e, f"{path}[{k!r}]")
        elif type(v).__module__.startswith(pkg_name) and hasattr(v, "__dict__"):
            for k, e in vars(v).items():
                walk(e, f"{path}.{k}")

    for path, v in root:
        walk(v, path)
    return [p for p, t in loose if t.untyped_storage().data_ptr() not in held], len(held)


def cache_roots(model, pkg_name):
    """The model's state outside parameters and buffers, and the package modules' module-level containers."""
    skip = {"_parameters", "_buffers", "_modules"}
    roots = [(f"{name or 'model'}.{k}", v) for name, mod in model.named_modules() for k, v in vars(mod).items()
             if k not in skip]
    for mname, mod in list(sys.modules.items()):
        if mname.startswith(pkg_name + ".") and mod is not None:
            roots += [(f"{mname}.{k}", v) for k, v in vars(mod).items() if isinstance(v, (dict, list))]
    return roots


def test_every_cached_tensor_is_ordered(pkg, oracle, env):
    """After forwards that fill every cache (eager fp16 at a cached resolution, a captured graph, fp32, NIQE), every
    CUDA tensor kept between calls is held under streams.Produced; a plain dict of tensors is caught."""
    from grl_image_restoration_b200 import metrics

    name = pkg.__name__
    m = micro_model(pkg, oracle, "fp16")
    x = x_at(51, R2)
    m(x)
    m.use_cuda_graph = True
    m(x)
    m.use_cuda_graph = False
    m.set_precision("fp32")
    m(x)
    m.set_precision("fp16")
    metrics.niqe_features(rand(52, 1, 3, 96, 96), NIQE_PARAMS, 0)
    torch.cuda.synchronize()
    loose, n = unordered_tensors(cache_roots(m, name), name)
    assert not loose, f"cached CUDA tensors outside the stream ordering: {loose[:10]}"
    assert n > 0 and m._graphs and m._table_cache and metrics._niqe_cache
    m._probe = {"t": torch.zeros(4, device="cuda")}
    loose, _ = unordered_tensors(cache_roots(m, name), name)
    assert loose == ["model._probe['t']"], loose
