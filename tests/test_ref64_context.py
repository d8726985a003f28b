"""oracle/ref64_context.py on a float32 stand-in ctx built from the reference: the unmutated stand-in passes every check,
and each plausible materialisation bug, applied to the stand-in, is flagged by the check named for it."""
import numpy as np
import pytest

from oracle import ref64
from oracle import ref64_context as X
from oracle import ref64_stages as S

F = np.float32


def _state(scene, kw=0, kg=0, shift_boundary=None):
    r = F(S.R)
    vdef = F(r * r * r * F(8.0 * 0.8))
    fluids = [dict(positions=f["positions"], density0=f["density0"], memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF),
                   volumes=np.full(len(f["positions"]), vdef, F) if f.get("volumes") is None else np.asarray(f["volumes"], F))
              for f in scene["fluids"]]
    bds = [dict(positions=b["positions"], velocities=b["velocities"], memberships=b.get("memberships", 1), filter=b.get("filter", 0xFFFFFFFF))
           for b in scene["boundaries"]]
    st = X.State(S.R, fluids, bds, kw, kg)
    bv = (1.0 / st.passes().boundary_volume_sum().value).astype(F)
    for b, (lo, hi) in zip(bds, zip(st.offsets(bds)[:-1], st.offsets(bds)[1:])):
        b["volumes"] = bv[lo:hi]
    return st


def _expect(st, fluid, rng):
    n = len(st.fluids[fluid]["positions"])
    ps = st.passes()
    fo = st.offsets(st.fluids)
    rows = slice(fo[fluid], fo[fluid + 1])
    return dict(velocities=rng.normal(0, 0.2, (n, 3)).astype(F), densities=rng.uniform(900, 1100, n).astype(F),
                volumes=st.fluids[fluid]["volumes"], acc_in=rng.normal(0, 1, (n, 3)).astype(F), counts_ff=ps.nf[rows],
                counts_fb=ps.nb[rows], handle=fluid, density0=st.fluids[fluid]["density0"], particle_radius=S.R, h=ps.h, contacts=True,
                boundaries=True, boundary_n=[len(b["positions"]) for b in st.boundaries])


def _standin(st, fluid, ex, boundaries=None):
    return X.standin(st, fluid, ex["velocities"], ex["densities"], ex["acc_in"], boundaries=boundaries)


_STATES = {}


def _get(name, kw=0, kg=0):
    key = (name, kw, kg)
    if key not in _STATES:
        _STATES[key] = _state(S.SCENES[name](), kw, kg)
    return _STATES[key]


@pytest.mark.parametrize("name,kw,kg", [("block", 0, 0), ("pairs", 0, 0), ("two_fluids", 0, 0), ("block", 1, 2), ("pairs", 3, 1)])
def test_the_unmutated_standin_passes(name, kw, kg):
    st = _get(name, kw, kg)
    for f in range(len(st.fluids)):
        ex = _expect(st, f, np.random.default_rng(f))
        rep = X.check(_standin(st, f, ex), st, f, ex)
        assert not rep.flagged(), rep.flagged()
        assert {"ff_weight", "ff_gradient", "fb_weight", "fb_gradient", "boundary_volume"} <= set(rep.worst)
        assert {"ff_csr", "ff_membership", "ff_self", "fb_membership", "positions", "densities", "acc_in", "boundary_views"} <= set(rep.bad)


def _rebuild(c, keep):
    """The contact list with only the entries `keep`, offsets recounted."""
    n = len(c["offsets"]) - 1
    i_of = np.repeat(np.arange(n), np.diff(c["offsets"]))
    out = {k: v[keep] for k, v in c.items() if k != "offsets"}
    out["offsets"] = np.r_[0, np.cumsum(np.bincount(i_of[keep], minlength=n))].astype(np.int64)
    return out


def _i_of(c):
    return np.repeat(np.arange(len(c["offsets"]) - 1), np.diff(c["offsets"]))


def _unzeroed_cubic(x, h):
    r = np.sqrt((x * x).sum(1))
    q = r / h
    d6 = 6.0 * 8.0 / (np.pi * h ** 3) / h
    return ((3.0 * q - 2.0) * q * d6 / np.where(r > 0, r, 1.0))[:, None] * x


# (mutant, scene, kernels, fluid) -> the checks that must flag it
MUTANTS = {
    "gradient_sign_flipped": (("block", 0, 0), 0, {"ff_gradient", "fb_gradient"}),
    "gradient_from_density_kernel": (("block", 1, 2), 0, {"ff_gradient", "fb_gradient"}),
    "weight_from_gradient_kernel_kind": (("block", 1, 2), 0, {"ff_weight", "fb_weight"}),
    "j_global_past_first_fluid": (("two_fluids", 0, 0), 0, {"ff_membership"}),
    "j_model_of_i_for_every_contact": (("two_fluids", 0, 0), 0, {"ff_membership"}),
    "boundary_j_model_off_by_one": (("two_fluids", 0, 0), 0, {"fb_membership"}),
    "self_contact_dropped": (("block", 0, 0), 0, {"ff_self", "ff_csr", "ff_membership"}),
    "entries_32_up_dropped": (("block", 0, 0), 0, {"ff_csr", "ff_membership"}),
    "offsets_shifted_by_one": (("block", 0, 0), 0, {"ff_csr", "ff_membership"}),
    "no_zeroing_below_1e-5_h": (("pairs", 0, 0), 0, {"ff_gradient"}),
    "densities_in_sorted_order": (("block", 0, 0), 0, {"densities"}),
    "boundary_views_one_pose_stale": (("block", 0, 0), 0, {"boundary_views", "fb_weight", "fb_gradient"}),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_each_materialisation_bug_is_flagged_by_name(mutant):
    (name, kw, kg), f, want = MUTANTS[mutant]
    st = _get(name, kw, kg)
    ex = _expect(st, f, np.random.default_rng(5))
    h = float(F(st.passes().h))
    if mutant == "boundary_views_one_pose_stale":   # the views of the pose before: the collider moved by 0.2 r since
        stale = [dict(b, positions=(np.asarray(b["positions"], F) - F(0.01)).astype(F)) for b in st.boundaries]
        cap = _standin(st, f, ex, boundaries=stale)
    else:
        cap = _standin(st, f, ex)
    ff, fb = cap["ff"], cap["fb"]
    if mutant == "gradient_sign_flipped":
        ff["gradient"], fb["gradient"] = -ff["gradient"], -fb["gradient"]
    elif mutant == "gradient_from_density_kernel":
        for c in (ff, fb):
            x = X.reference_contacts(st, f, "ff" if c is ff else "fb")[3]
            g = ref64.kernel(kw, "g", np.sqrt((x * x).sum(1)), h)[0]
            c["gradient"] = (np.where((x * x).sum(1) <= ref64.grad_threshold(kw, h), 0.0, g)[:, None] * x).astype(F)
    elif mutant == "weight_from_gradient_kernel_kind":
        for c in (ff, fb):
            x = X.reference_contacts(st, f, "ff" if c is ff else "fb")[3]
            c["weight"] = ref64.kernel(kg, "w", np.sqrt((x * x).sum(1)), h)[0].astype(F)
    elif mutant == "j_global_past_first_fluid":
        fo = st.offsets(st.fluids)
        ff["j"] = (ff["j"].astype(np.int64) + fo[ff["j_model"].astype(np.int64)]).astype(np.uint32)
        assert (ff["j_model"] > 0).any()
    elif mutant == "j_model_of_i_for_every_contact":
        assert (ff["j_model"] != f).any()
        ff["j_model"][:] = f
    elif mutant == "boundary_j_model_off_by_one":   # slot 1 reused, its contacts reported as slot 0's
        assert (fb["j_model"] == 1).any()
        fb["j_model"] = np.where(fb["j_model"] >= 1, fb["j_model"] - 1, fb["j_model"]).astype(np.uint32)
    elif mutant == "self_contact_dropped":
        i = _i_of(ff)
        cap["ff"] = _rebuild(ff, ~((ff["j_model"] == f) & (ff["j"] == i)))
    elif mutant == "entries_32_up_dropped":
        i = _i_of(ff)
        rank = np.arange(len(i)) - ff["offsets"][i]
        assert (rank >= 32).any()
        cap["ff"] = _rebuild(ff, rank < 32)
    elif mutant == "offsets_shifted_by_one":
        ff["offsets"] = np.r_[0, ff["offsets"][2:], ff["offsets"][-1]]
    elif mutant == "no_zeroing_below_1e-5_h":
        x = X.reference_contacts(st, f, "ff")[3]
        d2 = (x * x).sum(1)
        band = (d2 > ref64.EPS32 ** 2) & (d2 <= (1e-5 * h) ** 2)
        assert band.any()
        ff["gradient"][band] = _unzeroed_cubic(x[band], h).astype(F)
    elif mutant == "densities_in_sorted_order":
        cell = np.floor(np.asarray(cap["positions"], np.float64) / h).astype(np.int64)
        cap["densities"] = cap["densities"][np.lexsort(cell.T[::-1])]
    rep = X.check(cap, st, f, ex)
    assert want <= set(rep.flagged()), (mutant, rep.flagged(), rep.worst)


def test_additions_on_another_fluids_rows_are_flagged():
    """Accelerations out: the plugin of fluid 1 adds its pattern, written back at fluid 0's offset (the import's row range)
    instead of its own; and a correct write-back passes."""
    st = _get("two_fluids")
    rng = np.random.default_rng(3)
    twin = [rng.normal(0, 1, (len(fl["positions"]), 3)).astype(F) for fl in st.fluids]
    f = 1
    entry, add = twin[f], X.pattern(len(twin[f]), f)
    good = [t if k != f else (entry + add).astype(F) for k, t in enumerate(twin)]
    assert not X.check_acc_out(good, twin, entry, add, f).flagged()
    wrong = [t.copy() for t in twin]
    n = min(len(twin[0]), len(entry))
    wrong[0][:n] = (entry + add).astype(F)[:n]
    assert set(X.check_acc_out(wrong, twin, entry, add, f).flagged()) == {"acc_out"}
    # a plugin that adds nothing leaves every fluid as the twin's, and the check sees the missing addition
    assert "acc_out" in X.check_acc_out(twin, twin, entry, add, f).flagged()


def test_flags_and_scalars_are_checked():
    st = _get("block")
    ex = _expect(st, 0, np.random.default_rng(1))
    cap = _standin(st, 0, ex)
    assert not X.check(cap, st, 0, ex).flagged()
    for key, val in (("kernel_radius", F(0.2001)), ("density0", F(999.0)), ("fluid_index", 1), ("boundaries", None), ("ff", None)):
        bad = dict(cap, **{key: val})
        if key == "ff":
            bad["fb"] = None
        assert "scalars" in X.check(bad, st, 0, ex).flagged(), key
    off = dict(ex, contacts=False, boundaries=False)
    assert "scalars" in X.check(cap, st, 0, off).flagged()
    assert not X.check(dict(cap, ff=None, fb=None, boundaries=None), st, 0, off).flagged()
