"""The bookkeeping of a checking launcher, its case loader and a listing recorder, shared by test_gpu_tc_replay.py (the
tensor-core forward) and test_gpu_f32_replay.py (the fp32 forward).  A subclass (also a tc.Device) maps every kernel wrapper the forward launches
through to a method name m in `methods`, and gives `_outs_m` (the tensors the launch writes) and `_check_m` (its checks,
run after the launch has finished).  `run` checksums every written buffer right after its launch and re-verifies the sum
when a later launch reads it, so a stray write into a live neighbouring allocation fails; a wrapper without a checker
fails the run.  Like support.py, nothing here imports the product package."""
import weakref

import torch

import command_cases as CC
import grl_oracle as O
from support import build, dm_model, native_model, zoo_model

MAX_WINDOWS = 16  # attention windows checked per launch outside the first and last block of a stage
GEOMETRIES = 4    # attention geometries a replay keeps (a block's three passes, and the next block's first)


def _base(t):
    return t if t._base is None else t._base


def _checksum(t):
    w = t.reshape(-1).view({2: torch.int16, 4: torch.int32}[t.element_size()])
    return torch.stack([w.sum(dtype=torch.int64), w[::2].sum(dtype=torch.int64)])


def _tensors(v):
    if isinstance(v, torch.Tensor):
        yield v
    elif isinstance(v, (tuple, list)):
        for e in v:
            yield from _tensors(e)


def replay_case(pkg, oracle, cases, golden_loader, device, name):
    """(model, input, rggb) of a replay case "kind:what-precision": native:<shape> on "spread" weights, zoo:<golden>,
    dm:<golden> through the packed-Bayer head, micro:<case>[@HxW] on "routed" weights (at its own size or H x W),
    command:<checkpoint>@<H>x<W> (command_cases.py: a released checkpoint at the size its test command runs)."""
    kind, _, rest = name.partition(":")
    rest, precision = rest.rsplit("-", 1)
    if kind == "command":
        m, x, rggb = CC.model_and_input(pkg, oracle, CC.BY_NAME[f"command:{rest}"], device, precision)
        return m, x.to(device), rggb
    if kind == "native":
        m, x, _ = native_model(pkg, oracle, rest, "spread", device, precision)
        return m, x.to(device), False
    if kind == "zoo":
        m, gold = zoo_model(pkg, oracle, rest, device, precision)
        return m, torch.from_numpy(gold["x"]).to(device), False
    if kind == "dm":
        m = dm_model(pkg, oracle, device, precision)
        return m, golden_loader(f"dm_{rest}.npz")["cfa4"].to(device), True
    mname, _, size = rest.partition("@")
    c = cases[mname]
    hw = tuple(int(v) for v in size.split("x")) if size else c["hw"]
    m = build(pkg, oracle, c["cfg"], device, precision, style="routed")
    x = oracle.synth_input((c["batch"], c["cfg"]["in_channels"], *hw), seed=1234, noise_sigma=c["sigma"])
    return m, x.to(device), False


class Recorder:
    """A listing launcher (tc.Listing's protocol: nothing runs, no constant is cached) that records every wrapper a
    forward launches through, with the name of its first launch."""
    caches = False

    def __init__(self):
        self.fns = {}

    def listed(self, name, fn, *a, **kw):
        self.fns.setdefault(fn, name)

    def run(self, fn, *a, **kw):
        self.fns.setdefault(fn, getattr(fn, "__qualname__", repr(fn)))


class ReplayBase:
    """Results: `worst` {family: (statistic, gate, where)}, `failures` [(family, where, detail)], `mutations` {name:
    [caught, applied]}, `below` {name: blocks where it does not move the reference past twice the gate}.  With `poison`,
    every output is filled with NaN before its launch and must be finite after it (an element the kernel never writes
    fails)."""
    methods = {}
    poison = False

    def __init__(self, model, mutations, mutate=True, seed=0):
        self.model = model
        self.mutate, self.seed = mutate, seed
        self.owner = {}  # id(logit_scale / attn_transform) -> block name
        self.blocks = {}
        for si, layer in enumerate(model.layers):
            for bi, blk in enumerate(layer.blocks):
                name = f"stage{si}.block{bi}"
                self.blocks[name] = (blk, si, bi, len(layer.blocks))
                wa, sa = blk.attn.window_attn, blk.attn.stripe_attn
                for m in (wa.attn_transform, sa.attn_transform1, sa.attn_transform2):
                    self.owner[id(m)] = name
                self.owner[id(wa.attn_transform.logit_scale)] = name
        self.block, self.prev = None, None  # names of the current and the previous block
        self.saved = {}  # block name -> what the mutation controls take from the previous block
        self.sums = {}   # base data_ptr -> (weakref to the base, checksum, writer)
        self.worst, self.failures = {}, []
        self.mutations = {m: [0, 0] for m in mutations}
        self.below = {}
        self.geometries = {}  # (gq, gk, use_mask) -> grl_oracle.attn_pair_geometry, the GEOMETRIES latest

    # ---- bookkeeping ------------------------------------------------------------------------------
    def _gate(self, family, stat, gate, ok, where, detail=""):
        w = self.worst.get(family)
        if w is None or stat > w[0]:
            self.worst[family] = (stat, gate, where)
        if not ok:
            self.failures.append((family, where, f"{stat} (gate {gate}) {detail}"))

    def _exact(self, family, ok, where):
        self._gate(family, 0.0 if ok else 1.0, "bitwise", ok, where)

    def _check_reads(self, tensors, where):
        for t in tensors:
            b = _base(t)
            e = self.sums.get(b.data_ptr())
            if e is not None and e[0]() is b and not torch.equal(_checksum(b), e[1]):
                self.failures.append(("integrity", where, f"a buffer {e[2]} wrote changed before this launch read it"))

    def _record_writes(self, tensors, where):
        for t in tensors:
            b = _base(t)
            self.sums[b.data_ptr()] = (weakref.ref(b), _checksum(b), where)

    def _set_block(self, name):
        if name != self.block:
            self.prev, self.block = self.block, name
            self.saved = {k: v for k, v in self.saved.items() if k == self.prev}
            self._block_changed()

    def _block_changed(self):
        pass

    def _blk(self):
        return self.blocks[self.block][0]

    def _full_windows(self):
        _, _, bi, n = self.blocks[self.block]
        return bi == 0 or bi == n - 1

    def _mutation_here(self):
        """Mutation controls run at the first and last block of each stage that have a previous block."""
        return self.mutate and self.prev is not None and self._full_windows()

    def _mut(self, name, caught):
        self.mutations[name][1] += 1
        self.mutations[name][0] += bool(caught)
        if not caught:
            self.failures.append(("mutation", self.block, f"'{name}' passes its gate"))

    def _below(self, name):
        self.below[name] = self.below.get(name, 0) + 1

    def _geometry(self, gq, gk, use_mask):
        """grl_oracle.attn_pair_geometry of a launch, kept for the next launches of the replay: a whole-frame stripe
        mask is over a GB and takes seconds to build on the host, and every block uses its geometries several times."""
        key = (tuple(gq), tuple(gk), bool(use_mask))
        g = self.geometries.pop(key, None)
        if g is None:
            g = O.attn_pair_geometry(*key)
        self.geometries[key] = g  # most recent last
        while len(self.geometries) > GEOMETRIES:
            self.geometries.pop(next(iter(self.geometries)))
        return g

    def _windows(self, Bw):
        """Window indices to check: all of them in the first and last block of a stage, else the first, the last and
        MAX_WINDOWS - 2 seeded others."""
        if self._full_windows() or Bw <= MAX_WINDOWS:
            return torch.arange(Bw)
        g = torch.Generator().manual_seed(self.seed * 7919 + sum(map(ord, self.block)))
        mid = 1 + torch.randperm(Bw - 2, generator=g)[:MAX_WINDOWS - 2]
        return torch.cat([torch.tensor([0, Bw - 1]), mid]).sort().values

    # ---- the launcher -----------------------------------------------------------------------------
    def listed(self, name, fn, *args, **kw):
        self.run(fn, *args, _name=name, **kw)

    def run(self, fn, *args, _name=None, **kw):
        method = self.methods.get(fn)
        if method is None:
            raise AssertionError(f"{type(self).__name__} has no checker for {getattr(fn, '__qualname__', fn)}")
        outs = getattr(self, f"_outs_{method}")(*args, **kw)
        ins = [t for t in _tensors(list(args) + list(kw.values())) if all(t is not o for o in outs)]
        where = _name or (f"{self.block}:{method}" if self.block else method)
        self._check_reads(ins, where)
        if self.poison:
            for o in outs:
                o.fill_(float("nan"))
        fn(*args, **kw)
        torch.cuda.synchronize()
        if self.poison:
            self._exact("every output element written", all(bool(o.isfinite().all()) for o in outs), where)
        getattr(self, f"_check_{method}")(*args, _name=_name, **kw)
        self._record_writes(outs, where)

    # ---- report -----------------------------------------------------------------------------------
    def report(self, label, seconds, peak, extra=""):
        lines = [f"\n[replay] {label}: {seconds:.1f} s, peak memory {peak / 2 ** 30:.2f} GiB{extra}"]
        for fam, (s, gate, where) in sorted(self.worst.items()):
            lines.append(f"  {fam}: worst {s:.4g} (gate {gate}) at {where}")
        for name, (c, n) in self.mutations.items():
            lines.append(f"  mutation '{name}': fails its gate {c} / {n}"
                         + (f" ({self.below[name]} more below twice the gate)" if name in self.below else ""))
        for f in self.failures[:40]:
            lines.append(f"  FAIL {f}")
        print("\n".join(lines))
