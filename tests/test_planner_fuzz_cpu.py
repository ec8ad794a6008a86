"""Randomised initialisation programs through the whole host side, without a GPU.

Each program is what a module constructor might do to one tensor -- a factory (`empty/zeros/ones/
full/randn/rand`), an initialiser (`uniform_/normal_/fill_/trunc_normal_/kaiming_uniform_/
xavier_normal_`), then up to four of: in-place arithmetic, re-initialisation, writes through row and
slice views, out-of-place affine maps, `clone/detach`, casts to a 16-bit dtype and back, no-op casts.
The planner's verdict goes through `InitPlan` and the stream restatement
(tests/test_plan_oracle_cpu.py) and is compared with the same program run eagerly: constants and
by-value tensors bit for bit, RNG segments T1 (SURVEY.md 8c tolerances; a clamp that keeps a far tail
is judged by the distribution test alone).  Programs the planner cannot fold are counted, not failed:
they replay through ATen like everything does in the reference (deferred_init.cc:256-272).

The seeds are fixed, so the run is deterministic.  This harness found, in its first 150 programs,
(a) constants shared between the segments of a split tensor being written in place by an op meant
for one of them, (b) `x.to(dtype_it_already_has)` / `Model().float()` knocking tensors off the fused
path, (c) plans embedding one frozen sample of a program whose random draw sits in a dependency; and, in the
linked scripts, (d) the replay engine skipping in-place writes that were recorded on a tensor after an
early replay had already built it."""
import math
import os
import random

import pytest
import torch
from torch import nn

import test_plan_oracle_cpu as T
from oracle import tdx_oracle as O
from torchdistx_b200.deferred_init import deferred_init, plan_report
from torchdistx_b200.plan import InitPlan

# TDX_FUZZ_SCALE=20 runs twenty times the seeds (the defaults keep the CPU suite at a couple of minutes)
SCALE = max(1, int(os.environ.get("TDX_FUZZ_SCALE", "1")))

from oracle.fuzz_programs import (COLS, CONSTS, ROWS, VIEW_STEPS, Cell, Holder, LinkedHolder, apply_step,  # noqa: F401
                                  gen_cell, gen_linked, gen_program, gen_view_program, run_linked, run_program)


def run_seed(seed):
    r = random.Random(seed)
    progs = [gen_program(r) for _ in range(1 if seed % 3 else 2)]
    try:
        plan = InitPlan.from_module(deferred_init(Holder, progs))
    except ValueError as e:
        assert "random initialisation program the planner cannot fold" in str(e)
        return "replayed"
    got = O.evaluate_plan(plan, T.SEED, T.OFFSET)[0]
    torch.manual_seed(seed)
    own = T.named(Holder(progs))
    # (a regression net over ~1500 statistical checks, not the parity claim: SURVEY's bounds are 3.5
    # standard deviations of the difference and would fire by chance about once per run; x1.5 and
    # alpha = 1e-6 leave the gross errors a folding bug makes -- a wrong factor, offset, range, order)
    T.compare_with_eager(plan, got, own, own, clamps_by_ks_only=True, scale=1.5, alpha=1e-6)
    return "fused" if all(e.source != "value" for e in plan.entries) else "by value"


def test_random_init_programs_fold_to_what_eager_computes():
    seen = {"fused": 0, "replayed": 0, "by value": 0}
    for seed in range(600 * SCALE):
        try:
            seen[run_seed(seed)] += 1
        except AssertionError as e:
            raise AssertionError(f"seed {seed}: {e}") from e
    # most programs of this vocabulary fold (sub_/neg_/div_ on random tensors are what does not)
    assert seen["fused"] >= 350 * SCALE and seen["fused"] + seen["replayed"] + seen["by value"] == 600 * SCALE, seen


def test_writes_through_views_copies_and_shards():
    """The same, with writes through every kind of view (rows, slices, flat ranges: segments; columns,
    transposes: the planner must step back, not fold), `copy_` from constant / random / expanded
    sources, 0-dim tensor operands -- and every plan cut three ways: the shards concatenate to the whole."""
    seen = {"fused": 0, "replayed": 0, "by value": 0}
    for seed in range(500 * SCALE):
        r = random.Random(10_000 + seed)
        progs = [gen_view_program(r)]
        try:
            plan = InitPlan.from_module(deferred_init(Holder, progs))
        except ValueError as e:
            assert "random initialisation program the planner cannot fold" in str(e)
            seen["replayed"] += 1
            continue
        got, end, _ = O.evaluate_plan(plan, T.SEED, T.OFFSET)
        torch.manual_seed(seed)
        own = T.named(Holder(progs))
        try:
            T.compare_with_eager(plan, got, own, own, clamps_by_ks_only=True, scale=1.5, alpha=1e-6)
        except AssertionError as e:
            raise AssertionError(f"seed {seed}: {e}") from e
        parts = [O.evaluate_plan(plan, T.SEED, T.OFFSET, shard=(rank, 3))[:2] for rank in range(3)]
        assert all(p[1] == end for p in parts), seed
        for name, t in got.items():
            cat = torch.cat([p[0][name] for p in parts])
            assert torch.equal(cat.reshape(-1).view(torch.uint8), t.reshape(-1).view(torch.uint8)), (seed, name)
        seen["fused" if all(e.source != "value" for e in plan.entries) else "by value"] += 1
    assert seen["fused"] >= 120, seen


def row_relations(a, b):
    """Per row: do the two tensors hold the same draws?  1 = affinely tied (|correlation| of the 16
    columns > 0.9999: a clone, a copy, c * x + d of it), 0 = not, -1 = the row is constant in either."""
    a, b = a.double(), b.double()
    out = []
    for i in range(a.shape[0]):
        if a[i].std() == 0 or b[i].std() == 0 or not (torch.isfinite(a[i]).all() and torch.isfinite(b[i]).all()):
            out.append(-1)
        else:
            out.append(int(abs(torch.corrcoef(torch.stack([a[i], b[i]]))[0, 1].item()) > 0.9999))
    return out


def test_tensors_derived_from_each_others_intermediate_states():
    """`b = a.clone()` taken BEFORE `a.mul_(2)`, `b.copy_(a)` over b's own dead draw, casts and affine
    maps of a state that is then overwritten...: besides each tensor's own distribution, WHICH rows of
    two tensors hold the same random draws must be exactly what the eager run shows (a clone that got a
    fresh stream, or two tensors that got the same one, changes the pattern; no statistics involved)."""
    compared = tied = 0
    for seed in range(500 * SCALE):
        r = random.Random(20_000 + seed)
        progs, links = gen_linked(r)
        try:
            plan = InitPlan.from_module(deferred_init(LinkedHolder, progs, links))
        except ValueError as e:
            assert "random initialisation program the planner cannot fold" in str(e)
            continue
        got = O.evaluate_plan(plan, T.SEED, T.OFFSET)[0]
        torch.manual_seed(seed)
        own = T.named(LinkedHolder(progs, links))
        try:
            T.compare_with_eager(plan, got, own, own, clamps_by_ks_only=True, scale=1.5, alpha=1e-6)
        except AssertionError as e:
            raise AssertionError(f"seed {seed}: {e}") from e
        if any(st[0] in ("clamp", "data_clamp") for p in progs for st in p):
            continue  # (a clamp unties a row or not depending on the VALUES drawn: no exact pattern to compare)
        names = sorted(got)
        for x in range(len(names)):
            for y in range(x + 1, len(names)):
                if not (got[names[x]].dtype == got[names[y]].dtype == torch.float32):
                    continue  # (16-bit values are tied to their source only up to rounding: judged per tensor above)
                mine = row_relations(got[names[x]], got[names[y]])
                eager = row_relations(own[names[x]].detach(), own[names[y]].detach())
                # rows that are constant on either side carry no relation
                pairs = [(m, e) for m, e in zip(mine, eager) if m >= 0 and e >= 0]
                assert all(m == e for m, e in pairs), (seed, names[x], names[y], mine, eager)
                compared += len(pairs)
                tied += sum(e for _, e in pairs)
    assert compared > 5000 and tied > 500, (compared, tied)


DETERMINISTIC = {"reinit_u": "slice_fill", "reinit_n": "zero", "slice_normal": "slice_mul", "flat_normal": "flat_fill",
                 "copy_from_rng": "copy_from_const", "narrow_uniform": "reshape_fill", "select_col_normal": "col_zero"}


def test_replay_engine_in_any_materialisation_order():
    """The op-by-op engine itself (every CPU tensor, every program the planner cannot fold; reference
    deferred_init.cc:506-667): linked scripts with the random draws taken out, tensors materialised one
    by one in a RANDOM order -- bit for bit the eager result whatever the order (which ops a tensor's
    history needs, readers of intermediate states, in-place writes through views that were recorded
    after the value they change was already built)."""
    for seed in range(600 * SCALE):
        r = random.Random(30_000 + seed)
        progs, links = gen_linked(r)
        for p in progs:
            for _ in range(r.randint(0, 2)):
                b = r.randint(1, ROWS)
                p.insert(r.randint(1, len(p)), (r.choice(VIEW_STEPS), r.randint(0, b - 1), b, r.choice(CONSTS), r.choice(CONSTS),
                                                r.randint(0, COLS - 1)))
        for p in progs:
            for i, st in enumerate(p):
                if st[0] == "ctor" and st[1] in ("randn", "rand", "empty"):
                    p[i] = ("ctor", "full") + st[2:]
                elif st[0] == "init":
                    p[i] = ("init", "fill") + st[2:]
                elif st[0] in DETERMINISTIC:
                    p[i] = (DETERMINISTIC[st[0]],) + st[1:]
        links = {j: (i, min(cut, len(progs[i])), "copy_into_empty" if kind == "copy_into_rng" else kind, c, d, k)
                 for j, (i, cut, kind, c, d, k) in links.items()}
        from torchdistx_b200.deferred_init import materialize_tensor

        m = deferred_init(LinkedHolder, progs, links)
        order = [n for n, _ in m.named_parameters()]
        r.shuffle(order)
        got = {n: materialize_tensor(getattr(m, n)).detach() for n in order}
        eager = LinkedHolder(progs, links)
        for n in order:
            x, y = got[n], getattr(eager, n).detach()
            assert x.dtype == y.dtype and torch.equal(torch.nan_to_num(x.float()), torch.nan_to_num(y.float())) and \
                torch.equal(torch.isnan(x), torch.isnan(y)), (seed, n, order)


def test_parameter_data_and_module_idioms():
    """What model code does to a tensor once it is a Parameter: `p.data.normal_()`, `p.data[i].zero_()`,
    `p.data = p.data * c + d`, `with torch.no_grad(): p.mul_(c)`, `nn.init.*_(p)`, `requires_grad_(False)`,
    `module.to(dtype)` / `.float()` / `.to(device)` (real and no-op) -- HF `_init_weights` in short."""
    fused = 0
    for seed in range(500 * SCALE):
        r = random.Random(70_000 + seed)
        prog, steps = gen_cell(r)
        try:
            plan = InitPlan.from_module(deferred_init(Cell, prog, steps))
        except ValueError as e:
            assert "random initialisation program the planner cannot fold" in str(e)
            continue
        got = O.evaluate_plan(plan, T.SEED, T.OFFSET)[0]
        torch.manual_seed(seed)
        own = T.named(Cell(prog, steps))
        assert plan.entries[0].requires_grad == own["p"].requires_grad, seed
        try:
            T.compare_with_eager(plan, got, own, own, clamps_by_ks_only=True, scale=1.5, alpha=1e-6)
        except AssertionError as e:
            raise AssertionError(f"seed {seed}: {e}") from e
        fused += plan.entries[0].source != "value"
    assert fused >= 400, fused


class _Source(nn.Module):
    def __init__(self, prog):
        super().__init__()
        self.t = nn.Parameter(run_program(prog))


class _Reader(nn.Module):
    def __init__(self, src, kind, c, d, tail):
        super().__init__()
        s = src.detach()
        t = [lambda: s.clone(), lambda: s * c + d, lambda: torch.zeros_like(s).copy_(s), lambda: torch.cat([s[:5], s[5:]]) * 1.0][kind]()
        for st in tail:
            t = apply_step(t, st)
        self.u = nn.Parameter(t)


def test_tensors_that_read_an_earlier_recording():
    """`b = deferred_init(lambda: f(a))` with `a` from an EARLIER deferred_init, materialised in any
    order (a first; b first: a is then built on the spot as b's argument; b's tensor alone, then
    both modules): bit for bit the eager values, whatever a's program is."""
    from torchdistx_b200.deferred_init import materialize_module, materialize_tensor

    def deterministic(p):
        q = []
        for st in p:
            if st[0] == "ctor":
                st = ("ctor", "full" if st[1] in ("randn", "rand", "empty") else st[1], ROWS, COLS, st[4])
            elif st[0] == "init":
                st = ("init", "fill") + st[2:]
            elif st[0] in DETERMINISTIC:
                st = (DETERMINISTIC[st[0]],) + st[1:]
            if st[0] not in ("ctor", "init"):
                b = min(max(st[2], 1), ROWS)
                st = (st[0], min(st[1], b - 1), b) + st[3:5] + ((min(st[5], COLS - 1),) if isinstance(st[5], int) else (st[5],))
            q.append(st)
        return q

    for seed in range(400 * SCALE):
        r = random.Random(60_000 + seed)
        p1 = deterministic(gen_view_program(r) if r.random() < 0.5 else gen_program(r))
        tail = [st for st in deterministic(gen_program(r)) if st[0] not in ("ctor", "init")]
        kind, c, d = r.randrange(4), r.choice(CONSTS), r.choice(CONSTS)
        m1 = deferred_init(_Source, p1)
        m2 = deferred_init(_Reader, m1.t, kind, c, d, tail)
        order = r.choice(["source first", "reader first", "reader's tensor, then both"])
        if order == "source first":
            materialize_module(m1)
            materialize_module(m2)
        elif order == "reader first":
            materialize_module(m2)
            materialize_module(m1)
        else:
            u = materialize_tensor(m2.u)
            materialize_module(m1)
            materialize_module(m2)
            assert m2.u is u, seed
        e1 = _Source(p1)
        e2 = _Reader(e1.t, kind, c, d, tail)
        for mine, want in ((m1.t, e1.t), (m2.u, e2.u)):
            a, b = mine.detach(), want.detach()
            assert a.dtype == b.dtype and torch.equal(torch.nan_to_num(a.float()), torch.nan_to_num(b.float())), (seed, order, kind)


def test_the_c_abi_accepts_every_table_the_planner_emits():
    """`tdx_init_prepare` (host side of include/tdx_init.h: argument validation, tiling, work lists; no
    GPU involved) on the descriptor tables of random plans, whole and sharded, in all three dtypes:
    nothing the planner emits is outside what the kernels' ABI admits (source / dtype pairs, epilogue
    length, element alignment of every destination)."""
    from torchdistx_b200 import _cabi
    from torchdistx_b200.plan import assign_pass_offsets, entry_descriptors, shard_range

    checked = 0
    for seed in range(400 * SCALE):
        r = random.Random(90_000 + seed)
        progs = [gen_view_program(r) if r.random() < 0.5 else gen_program(r) for _ in range(r.randint(1, 3))]
        prev = torch.get_default_dtype()
        torch.set_default_dtype(r.choice([torch.float32, torch.bfloat16, torch.float16]))
        try:
            plan = InitPlan.from_module(deferred_init(Holder, progs))
        except ValueError:
            continue
        finally:
            torch.set_default_dtype(prev)
        for shard in (None, (1, 3)):
            descs, assigned, offset, base = [], {}, 8, 1 << 20
            for e in plan.entries:
                if e.source in ("alias", "value"):
                    continue
                begin, count, _ = shard_range(e, shard)
                passes, offset = assign_pass_offsets(e, assigned, offset)
                descs += entry_descriptors(e, base, begin, count, 1234, passes)
                base += ((count * 8 + 255) // 256 + 1) * 256
            if descs:
                assert _cabi.prepare(descs) > 0, (seed, shard)
                checked += 1
    assert checked >= 300, checked


def test_the_bugs_the_fuzzer_found_stay_fixed():
    # (a) a constant shared by the segments of a split tensor, written in place by an op meant for one
    def shared(which):
        t = torch.full((70, 16), -1.5)
        t = (t * -1.5 + -0.125).to(torch.bfloat16)
        if which == "row_then_all":
            t[23].zero_()
            t.add_(1.0)  # (added twice to the two outer segments)
        else:
            t[11:44].mul_(2.0)  # (doubled the whole tensor)
        return nn.ParameterList([nn.Parameter(t)])

    for which in ("row_then_all", "slice_only"):
        plan = InitPlan.from_module(deferred_init(shared, which))
        assert plan.entries[0].source == "const" and len(plan.entries[0].segments) == 3
        got = O.evaluate_plan(plan, T.SEED, T.OFFSET)[0]
        assert torch.equal(got["0"], shared(which)[0].detach()), which

    # (b) conversions that have nothing to convert return the tensor itself: still on the fused path
    for fn in (lambda: nn.Linear(16, 8).float(), lambda: nn.Linear(16, 8).to(torch.float32),
               lambda: nn.Linear(16, 8).to("cpu"), lambda: nn.Linear(16, 8).to(torch.bfloat16).to(torch.bfloat16),
               lambda: nn.ParameterList([nn.Parameter(torch.empty(8, 8).normal_().to(torch.float32))])):
        r = plan_report(deferred_init(fn))
        assert all(v["fusible"] and v["source"] in ("uniform", "normal") for v in r.values()), r

    # (d) the replay engine: `b = a.clone()` is replayed as part of a's history (it reads a); the write
    # through a view of b recorded after it must still run before `b * c + d` reads b
    def late_write():
        a = torch.ones(8, 4)
        b = a.clone()
        b[2:5].normal_(0.5, 3.0)
        m = nn.Module()
        m.a, m.b = nn.Parameter(a), nn.Parameter(b * -0.125 + -0.125)
        return m

    from torchdistx_b200.deferred_init import materialize_tensor

    for first in ("a", "b"):
        m = deferred_init(late_write)
        torch.manual_seed(0)
        out = {n: materialize_tensor(getattr(m, n)) for n in (("a", "b") if first == "a" else ("b", "a"))}
        torch.manual_seed(0)
        e = late_write()
        assert torch.equal(out["a"], e.a) and torch.equal(out["b"], e.b), first

    # (c) a random draw in a DEPENDENCY of an unfusable program is still a random program: not embedded
    def hidden():
        return nn.ParameterList([nn.Parameter(torch.sin(torch.randn(8, 8)) * 2.0 + 3.0)])  # (sin: not a foldable step)

    assert not plan_report(deferred_init(hidden))["0"]["fusible"]
    s0 = torch.get_rng_state()
    with pytest.raises(ValueError, match="random initialisation program the planner cannot fold"):
        InitPlan.from_module(deferred_init(hidden))
    assert torch.equal(torch.get_rng_state(), s0)  # (probed under a forked generator)
