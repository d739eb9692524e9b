"""undistort on remap tables the FOV model never produces (tests/remap_families.py), pinned on the CPU: the numpy statement
(undistort_spec), the plain-C restatement (oracle port: undistort and getImage) and, where oracle/_ref was built, the reference's
own compiled UndistorterFOV::undistort<uchar> / <float>, all bit for bit.  The reference object is built from a camera.txt with the
family's dimensions and its remapX / remapY are overwritten with the family's tables, which are all inside the domain D."""
import numpy as np
import pytest

import remap_families as RF
import undistort_spec as spec
from conftest import assert_bits_equal

F32 = np.float32
FAMILIES = sorted(RF.REGISTRY)


@pytest.fixture(scope="module")
def ref_undistort(tmp_path_factory):
    """(family) -> (u8 image -> output, f32 image -> output) through the reference's compiled undistort, or None without oracle/_ref."""
    from oracle import loader
    if not loader.ref_available():
        return None
    o = loader.RefOracle()
    root = tmp_path_factory.mktemp("ref_cams")

    def make(f):
        cam = root / f"{f.name}_{f.in_w}x{f.in_h}_{f.out_w}x{f.out_h}.txt"
        cam.write_text(f"0.5 0.5 0.5 0.5 0\n{f.in_w} {f.in_h}\ncrop\n{f.out_w} {f.out_h}\n")
        rf = o.fov(str(cam))
        assert rf.valid and (rf.in_w, rf.in_h, rf.out_w, rf.out_h) == (f.in_w, f.in_h, f.out_w, f.out_h)
        assert spec.in_domain(f.rx, f.ry, f.in_w, f.in_h).all()      # only tables inside D go into the reference object
        n = f.out_w * f.out_h
        np.ctypeslib.as_array(o.lib.oref_fov_remap_x(rf.h), (n,))[:] = f.rx
        np.ctypeslib.as_array(o.lib.oref_fov_remap_y(rf.h), (n,))[:] = f.ry
        return rf
    return make


@pytest.mark.parametrize("name", FAMILIES)
def test_spec_port_and_reference_agree(name, port, ref_undistort):
    f = RF.get(name)
    assert spec.in_domain(f.rx, f.ry, f.in_w, f.in_h).all(), f"{name}: entries outside D"
    n_in = f.in_w * f.in_h
    seed = sum(map(ord, name))
    img8 = RF.frame_u8(n_in, seed)
    imgf = RF.special_floats(n_in, seed + 1)
    rf = ref_undistort(f) if ref_undistort else None
    for img in (img8, imgf):
        s = spec.undistort(f.rx, f.ry, f.in_w, f.in_h, img)
        assert_bits_equal(port.undistort(f.rx, f.ry, f.in_w, img), s, f"{name} {img.dtype}: port vs spec")
        if rf is not None:
            assert_bits_equal(rf.undistort(img), s, f"{name} {img.dtype}: reference vs spec")
    # getImage through the port (unmap, then undistort<float>) against the spec, with extreme photometric tables
    ginv, vinv = RF.arbitrary_photometric(n_in, seed + 2)
    for flags in ((1, 0, 0, 0), (1, 1, 0, 0), (1, 1, 1, 1), (1, 0, 0, 1)):
        assert_bits_equal(port.get_image(f.rx, f.ry, f.in_w, f.in_h, ginv, vinv, img8, *flags),
                          spec.get_image(f.rx, f.ry, f.in_w, f.in_h, ginv, vinv, img8, *flags), f"{name} getImage flags={flags}")


def test_reference_was_compared_wherever_it_is_built(ref_undistort):
    """The bit-for-bit pin against the reference's own undistort runs wherever oracle/_ref exists."""
    from oracle import loader
    assert (ref_undistort is not None) == loader.ref_available()


def test_spec_states_truncation_and_black_rule():
    """Hand-worked entries: y in (-1, 0) keeps row 0 with a negative fraction (floor would pick row -1), -0.0 is a valid x, a NaN y
    under a negative x is black, and integer coordinates read one pixel."""
    img = np.arange(12, dtype=F32).reshape(3, 4) * 10        # 4 x 3 frame
    rx = np.array([1.0, 1.5, -0.0, -1e-45, -np.inf, 2.0], F32)
    ry = np.array([-0.5, 1.0, 0.0, np.nan, 7.0, 1.0], F32)
    out = spec.undistort(rx, ry, 4, 3, img.reshape(-1))
    # (1, -0.5): fx = 0, fy = -0.5 -> w2 = -0.5, w0 = 1.5: 1.5 * s(1,0) - 0.5 * s(1,1) = 15 - 25
    assert out[0] == F32(1.5) * 10 + F32(-0.5) * 50
    assert out[1] == F32(0.5) * 50 + F32(0.5) * 60        # (1.5, 1): s(1, 1) and s(2, 1)
    assert out[2] == 0 and not np.signbit(out[2]) and spec.in_domain(rx[2:3], ry[2:3], 4, 3).all()
    assert out[3] == 0 and out[4] == 0
    assert out[5] == 60                                      # (2, 1): s(2, 1) alone
    # outside D: x = W-1, y = H-1, y = -1, NaN x, NaN y under a valid x, +inf
    bad_x = np.array([3.0, 1.0, 1.0, np.nan, 1.0, np.inf], F32)
    bad_y = np.array([0.0, 2.0, -1.0, 0.0, np.nan, 0.0], F32)
    assert not spec.in_domain(bad_x, bad_y, 4, 3).any()


def test_plan_model_reaches_the_branches_each_family_exists_for():
    """The families reach, in the plan model, what they are built for; the GPU module checks the same on the library's own plan."""
    def m(name, g=8):
        return RF.plan_model(RF.get(name), g)
    assert m("scatter_1280x1024")["staged"] == 0 and m("scatter_black_1280x1024")["staged"] == 0
    assert m("to_40x30_1280x1024")["staged"] == 0
    assert RF.granularity_without_pitch_search(RF.get("many_classes_g16_1920x1080")) == 16
    assert RF.granularity_without_pitch_search(RF.get("many_classes_g32_1920x1080")) == 32
    # no plan has more than 64 classes at granularity 32 (so none is left without TMA by its class count): the staged limits leave
    # at most 40 (width, rounded height) pairs, counting for each pair its lowest box height bh8 - 31
    pairs32 = {(bw, bh8) for bw in range(16, 257, 16) for bh8 in range(32, 257, 32)
               if bw * bh8 <= RF.MAX_STAGED_PX
               and -(-(bh8 - 31) // max(1, RF.THREADS >> max(2, (bw - 1).bit_length() - 2))) <= RF.MAX_BOX_WORDS}
    assert len(pairs32) <= RF.MAX_CLASSES
    ramp = m("minify_ramp_1920x1080")
    assert ramp["staged"] > 0 and ramp["direct"] > 0
    cb = m("checkerboard_1280x1024")
    assert cb["staged"] > 0 and cb["direct"] > 0 and cb["empty"] > 0 and cb["black"] > cb["empty"]
    for name in ("identity_int_1280x1024", "edges_1280x1024", "subnormal_333x217", "magnify16_1280x1024", "rot90_1920x1080"):
        assert m(name)["staged"] > 0, name
