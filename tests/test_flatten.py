"""The flattening stage of tb200_problem_create (trajopt_b200/csrc/flatten.h) without a device: the folded robot, the
hatched cost and constraint lists, the kernel-order side tables, the term tables, the fixed variables and the banded
quadratic objective of each description hash to pinned FNV-1a digests.  These are the bytes the library uploads, so a
change to the flattening that alters any of them fails here on any machine.  The digests were taken from the library
as it was before the stage moved into its own header."""
import ctypes as C

import pytest

import cpp_host
from trajopt_b200 import capi, problems


@pytest.fixture(scope="module")
def flat(tmp_path_factory):
    lib = C.CDLL(cpp_host.build(tmp_path_factory, "flatten_digest", shared=True))
    lib.flatten_digest.argtypes = [C.POINTER(capi.ProblemDescC), C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
    lib.flatten_digest.restype = C.c_int
    return lib


def _descriptions():
    """name -> maker: configs[1]-[4] at two lengths each, the shape sweep, the reference's JSON files and configs[2]'s
    term variants (the description with fixed_dofs)."""
    from test_reference_json import NAMES, _load
    from test_shape_sweep import CASES, DESCS
    makers = {}
    for cfg, Ts in (("config1", (10, 30)), ("config2", (10, 30)), ("config3", (20, 50)), ("config4", (20, 40))):
        for T in Ts:
            makers[f"{cfg}_T{T}"] = lambda cfg=cfg, T=T: getattr(problems, cfg)(B=2, T=T)
    for name in CASES:
        makers[f"sweep_{name}"] = lambda name=name: DESCS[name]
    for name in NAMES:
        makers[f"json_{name}"] = lambda name=name: _load(name)
    makers["variants"] = lambda: problems.config_variants(B=2, T=10)
    return makers


DESCRIPTIONS = _descriptions()
PINNED = {
    "config1_T10": "30fd39ac9fe9f685",
    "config1_T30": "7d94ef0a50238e11",
    "config2_T10": "2a9ff0584cc81e59",
    "config2_T30": "2934c2415fb0a2ac",
    "config3_T20": "7c9dcd3508c27351",
    "config3_T50": "97b90652b33eda9b",
    "config4_T20": "2a05eeb728a95c6f",
    "config4_T40": "597d86aaf5aefdcb",
    "sweep_d7_T1": "27f98ce7095eaea8",
    "sweep_d7_T3": "e8e7e599f18dceea",
    "sweep_d7_T5": "f6df0d8ea1917a80",
    "sweep_d7_T7": "146b1d2f7e04c696",
    "sweep_d7_T15": "077b458e93b8cc6e",
    "sweep_d7_T16": "7e41da17345c87f6",
    "sweep_d7_T23": "3d4390d2f06cb446",
    "sweep_d7_T24": "74c7135a1e2db236",
    "sweep_d7_T25": "02e16ffe865cbdd8",
    "sweep_d7_T27": "5663c9dd57558c4a",
    "sweep_d7_T31": "7db58618bbd0d332",
    "sweep_d7_T33": "097b95c98c5ec110",
    "sweep_d7_T36": "2f4207a0bb50c172",
    "sweep_d7_T37": "d630643abc590778",
    "sweep_d7_T49": "b526d84e7642cb70",
    "sweep_d7_T59": "48f8081785596da6",
    "sweep_d7_T64": "a08f1e0f74dff416",
    "sweep_d7p_T5": "3eee742fe403d0fb",
    "sweep_d7p_T16": "8c2eb02bc02dfab2",
    "sweep_d7p_T24": "fe9dba8a852b6a4d",
    "sweep_d7p_T33": "a50876869ea0865c",
    "sweep_d7p_T64": "e39012496772b360",
    "sweep_d6_T3": "55434987686bca08",
    "sweep_d6_T9": "d049dea6ccd5946a",
    "sweep_d6_T16": "3e7f9eb09924d088",
    "sweep_d6_T24": "b31d98480f34be0c",
    "sweep_d6_T33": "ec252dc98e0121ea",
    "sweep_d6_T41": "c29773e730060636",
    "sweep_d3_T3": "534905c66af41a9c",
    "sweep_d3_T9": "a6164de04530133a",
    "sweep_d3_T16": "fed53936d79b5ca4",
    "sweep_d3_T24": "64632afde47c4adc",
    "sweep_d3_T33": "6ff47ac7b2db7ab6",
    "sweep_d3_T64": "7e91e47805aa010c",
    "sweep_d2_T2": "71f6fb02cee9157f",
    "sweep_d2p_T2": "944c15b208d88183",
    "sweep_d2_T13": "30f3810e6dcd796c",
    "sweep_d2p_T13": "39f4bee8cc937a30",
    "sweep_d2_T40": "99d51587e5a8b37e",
    "sweep_d2p_T40": "593245bf5a85a764",
    "sweep_d14_T3": "2efe3a739a9db77f",
    "sweep_d14_T9": "b7116d167dcd0c61",
    "sweep_d14_T17": "c6587a9d0b63e8d1",
    "sweep_d14_T50": "b4120876a0659665",
    "sweep_d14_T62": "ad37251a57868bdd",
    "sweep_d7_T12_crowded": "a039bdf3937b1c31",
    "sweep_d7_T10_obs64": "dda2884ced02fefb",
    "sweep_d7_T10_obs64_shared": "dda2884ced02fefb",
    "json_arm_around_table": "96da7031354692a1",
    "json_simple_collision_test": "ec8a0cd78a86687b",
    "json_numerical_ik1": "e04b2fa0b2cfec4d",
    "json_box_cast_test": "ac120f47b38fc3e6",
    "variants": "ce2c44951d7d05be",
}


@pytest.mark.parametrize("name", list(DESCRIPTIONS))
def test_flattened_description_is_pinned(flat, name):
    d = DESCRIPTIONS[name]()
    h = C.c_uint64()
    msg = C.create_string_buffer(256)
    rc = flat.flatten_digest(C.byref(d.c), C.byref(h), msg, len(msg))
    assert rc == 0, msg.value.decode()
    assert f"{h.value:016x}" == PINNED[name]


def test_flatten_reports_the_library_message(flat):
    d = problems.config2(B=2, T=10)
    d._terms[2].target_slot = 1
    msg = C.create_string_buffer(256)
    rc = flat.flatten_digest(C.byref(d.c), C.byref(C.c_uint64()), msg, len(msg))
    assert rc == capi.ERR_INVALID and msg.value.decode() == "cart_pose target_slot out of range"
