"""Refusals every match, LBR and agent creator makes before it touches a device: a null output pointer, and a seat with neither a
handle nor a blueprint.  Each returns CFRB_EINVAL (-1), names the entry point that was called, and leaves *out null."""
import ctypes as C

import pytest

from rebel_b200 import capi

I32, U64 = C.c_int32, C.c_uint64
NULL = C.c_void_p(None)
AVG, EN = capi.MATCH_AVERAGE, capi.MATCH_EVERY_NODE


def call(name, out):
    """Entry point `name` with an empty seat (no handle, no blueprint), writing to `out` (None: a null output pointer)."""
    L = capi.lib()
    o = C.byref(out) if out is not None else None
    empty = capi.MatchAgent(None, None, AVG)
    args = {
        "cfrb_match_create": (NULL, NULL, I32(8), I32(8), U64(0), I32(AVG), o),
        "cfrb_match_create2": (NULL, NULL, I32(8), I32(8), U64(0), I32(EN), I32(AVG), o),
        "cfrb_match_create3": (C.byref(empty), C.byref(empty), I32(8), I32(8), U64(0), o),
        "cfrb_match_create_lbr": (NULL, I32(8), I32(8), U64(0), o),
        "cfrb_match_create_lbr2": (NULL, I32(8), I32(8), U64(0), I32(EN), o),
        "cfrb_match_create_lbr_blueprint": (NULL, I32(8), I32(8), U64(0), o),
        "cfrb_agent_create": (NULL, I32(4), U64(0), I32(AVG), o),
        "cfrb_agent_create_blueprint": (NULL, I32(4), U64(0), o),
    }[name]
    return capi._check(getattr(L, name)(*args))


EMPTY_SEAT = {
    "cfrb_match_create": r"null handle \(local best response against one agent is cfrb_match_create_lbr",
    "cfrb_match_create2": r"null handle \(local best response against one agent is cfrb_match_create_lbr",
    "cfrb_match_create3": "an agent needs a handle or a blueprint",
    "cfrb_match_create_lbr": "null handle",
    "cfrb_match_create_lbr2": "null handle",
    "cfrb_match_create_lbr_blueprint": "null blueprint",
    "cfrb_agent_create": "null handle",
    "cfrb_agent_create_blueprint": "null blueprint",
}


@pytest.mark.parametrize("name", sorted(EMPTY_SEAT))
def test_null_output_is_refused(name):
    with pytest.raises(capi.CfrbError, match=f"^cfrb error -1: {name}: null argument"):
        call(name, None)


@pytest.mark.parametrize("name", sorted(EMPTY_SEAT))
def test_empty_seat_is_refused(name):
    out = C.c_void_p(1234)
    with pytest.raises(capi.CfrbError, match=f"^cfrb error -1: {name}: {EMPTY_SEAT[name]}"):
        call(name, out)
    assert not out.value


def test_create3_refuses_a_null_seat_pointer():
    out = C.c_void_p(1234)
    seat = capi.MatchAgent(None, None, AVG)
    for a, b in [(None, C.byref(seat)), (C.byref(seat), None)]:
        with pytest.raises(capi.CfrbError, match="^cfrb error -1: cfrb_match_create3: null argument"):
            capi._check(capi.lib().cfrb_match_create3(a, b, 8, 8, 0, C.byref(out)))
