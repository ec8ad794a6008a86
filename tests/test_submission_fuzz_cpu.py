"""Mixed submissions on the host: every table tests/submission_fuzz.py draws must prepare.

`tdx_init_prepare` validates a descriptor table and lays its plan out without a device (the host then
assumes 132 SMs).  Tables that span more kernel families than one plan header holds (47) are laid out
as consecutive plans in one workspace, so they must prepare like any other -- a model that mixes fp32,
bf16 and fp16 tensors, epilogues, casts and Shard(1) windows reaches more than 47 families.  The
prepared size must stay within tdx_init_workspace_bytes(n), the bound callers may allocate up front.

The routing restatement in submission_fuzz.py is checked here for what it claims about the forced
tables (the threshold, rider and family-count regimes really are on the side they are named for); the
GPU test holds the library's launch counts to it.
"""
import ctypes

import pytest

import submission_fuzz as F
from torchdistx_b200 import _cabi as C

SEEDS = 200
ARENA, SOURCE = 1 << 44, 1 << 43  # (nothing is written: any element-aligned addresses do)


def prepare(descs):
    lib = C.load()
    arr = (C.TdxInitDesc * len(descs))(*descs)
    need = ctypes.c_size_t(0)
    rc = lib.tdx_init_prepare(arr, len(descs), ctypes.byref(need))
    return rc, int(need.value), lib.tdx_last_error().decode()


def check_table(t):
    descs = t.descs(ARENA, SOURCE)
    rc, need, err = prepare(descs)
    assert rc == 0, f"{t.name}: {len(descs)} descriptors, {F.groups(t.specs)} families: error {rc}: {err}"
    assert need <= C.load().tdx_init_workspace_bytes(len(descs)), (t.name, need)
    assert (need == 0) == (not descs), (t.name, need)


@pytest.mark.parametrize("seed", range(SEEDS))
def test_every_table_prepares(seed):
    for t in F.tables(seed):
        check_table(t)


def test_the_row_order_is_the_library_family_count():
    # (80 rows: 30 in the base unit, 11 state-space, 20 window, 16 ATen, band, gather and sincos)
    assert len(F.ROW_ORDER) == 80


def test_a_table_of_every_row():
    t = F.every_row(__import__("numpy").random.default_rng(1))
    assert set(F.route(t.specs)) == set(F.ROW_ORDER)
    check_table(t)


@pytest.mark.parametrize("seed", range(8))
def test_forced_regimes_are_what_they_are_named(seed):
    seen = set()
    for t in F.tables(seed, n_random=0):
        fam = F.route(t.specs)
        lut = [f for f in fam if f[0] == "lut"]
        tag = t.tags[0]
        seen.add(tag)
        if tag == "table-below":
            assert not lut, t.name
        elif tag == "table-at":
            assert lut, t.name
        elif tag in ("riders-at", "riders-above"):
            ride = [f for f, s in zip(fam, t.specs) if s.kw["src"] in (C.TDX_SRC_CONST, C.TDX_SRC_IOTA)]
            assert all(f[0] == "lut" for f in ride) == (tag == "riders-at"), t.name
            host = sum(s.nbytes for f, s in zip(fam, t.specs) if f[0] == "lut" and s.kw["src"] not in
                       (C.TDX_SRC_CONST, C.TDX_SRC_IOTA))
            riders = sum(s.nbytes for s in t.specs if s.kw["src"] in (C.TDX_SRC_CONST, C.TDX_SRC_IOTA))
            assert riders * 16 - host == (0 if tag == "riders-at" else 16), t.name
        elif tag.startswith("preassigned"):
            # (every descriptor of the table group, riders included, counted as the library counts tiles)
            tiles = sum(F.tiles_of(s, ARENA + s.off, F.LUT_TILE_VECS) for f, s in zip(fam, t.specs) if f[0] == "lut")
            assert tiles == 16 * F.SM - (tag == "preassigned-below"), (t.name, tiles)
        elif tag == "static-grabs":
            per_sm, delta = map(int, t.name.split(":")[1].split("x"))
            direct = ("direct", F.N, C.TDX_BF16, C.TDX_ALGO_ICDF16, "none")
            tiles = sum(F.tiles_of(s, ARENA + s.off, 1024) for f, s in zip(fam, t.specs) if f == direct)
            assert tiles == F.STATIC_TILES_PER_CTA * F.SM * per_sm + delta, (t.name, tiles)
        elif tag == "families-47":
            assert F.groups(t.specs) == 47, t.name
        elif tag == "wide":
            assert F.groups(t.specs) > 47, t.name
    assert seen >= {"table-below", "table-at", "riders-at", "riders-above", "preassigned-below", "preassigned-at",
                    "static-grabs", "one", "families-47", "wide", "every-row"}


def test_one_plan_upload_still_takes_one_plan():
    """tdx_plan_upload keeps its documented limit: a table of more than 47 families is refused there with
    a message that names the call to use instead (nothing reaches the device: the plan is checked first)."""
    t = [x for x in F.tables(3, n_random=0) if x.name.endswith("families-48")][0]
    descs = t.descs(ARENA, SOURCE)
    lib = C.load()
    arr = (C.TdxInitDesc * len(descs))(*descs)
    plan = C.TdxPlan()
    rc = lib.tdx_plan_upload(arr, len(descs), None, 0, None, ctypes.byref(plan))
    assert rc == -1 and "tdx_init_launch" in lib.tdx_last_error().decode()
