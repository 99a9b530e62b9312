"""The Python binding against include/b200bt.h: every prototype's ctypes signature, every struct's host mirror and every
constant _lib.py restates.  No GPU and no built library: importing _lib does not load the shared object."""
import ctypes as C

import numpy as np
import pytest

import abi_header
from ai_crypto_trader_b200 import _lib, sweep

HEADER = abi_header.parse()
CTYPES = {"int": C.c_int, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "float": C.c_float, "double": C.c_double,
          "int64_t": C.c_int64, "uint64_t": C.c_uint64, "uint8_t": C.c_uint8, "unsigned char": C.c_ubyte, "char": C.c_char}

# header struct -> its host mirrors: a ctypes Structure, a numpy row dtype, or a tuple naming all-8-byte fields
STRUCT_MIRRORS = [
    ("b200bt_individual", _lib.Individual), ("b200bt_individual", sweep.INDIVIDUAL_DTYPE),
    ("b200bt_lane_stats", _lib.LANE_STATS_FIELDS), ("b200bt_sweep_config", _lib.SweepConfig),
    ("b200bt_bt_params", _lib.BtParams), ("b200bt_regime_params", _lib.RegimeParams),
    ("b200bt_regime_window", _lib.REGIME_WINDOW_DTYPE), ("b200bt_grid_individual", _lib.GridIndividual),
    ("b200bt_grid_regime_rule", _lib.GridRegimeRule), ("b200bt_grid_stats", _lib.GRID_STATS_FIELDS),
    ("b200bt_grid_service_stats", _lib.GRID_SERVICE_FIELDS), ("b200bt_dca_individual", _lib.DcaIndividual),
    ("b200bt_dca_stats", _lib.DCA_STATS_FIELDS), ("b200bt_dca_service", _lib.DCA_SERVICE_FIELDS),
    ("b200bt_rl_agent", _lib.RlAgent), ("b200bt_rl_agent_state", _lib.RL_STATE_DTYPE),
    ("b200bt_vp_params", _lib.VpParams), ("b200bt_vp_row", _lib.VP_ROW_DTYPE),
    ("b200bt_monitor_params", _lib.MonitorParams), ("b200bt_monitor_row", _lib.MONITOR_ROW_DTYPE),
]
# header structs the host builds without a mirror: sweep.ChunkPlan fills b200bt_chunk_item rows as int32 [n][4]
NO_HOST_MIRROR = {"b200bt_chunk_item": ("individual", "chunk", "n_chunks", "segment")}


def _constants():
    """(value _lib uses, the macro it mirrors) for every constant _lib.py restates."""
    pairs = [(_lib.ABI_VERSION, "B200BT_ABI_VERSION"), (0, "B200BT_OK"),                 # _lib.call: 0 is success
             (_lib.PRIMARY_ZERO, "B200BT_PRIMARY_ZERO"), (len(_lib.ANALYZER_COLUMNS), "B200BT_ANALYZER_COLUMNS"),
             (len(_lib.MM_COMBINATIONS), "B200BT_MM_COMBINATIONS"), (len(_lib.MM_LABEL_FIELDS), "B200BT_MM_LABEL_FIELDS")]
    pairs += [(getattr(_lib, name), "B200BT_" + name) for name in (
        "EVENT_EXIT", "EVENT_SELL", "EVENT_BAR_MASK", "GRID_ADAPT_REGIME", "GRID_AUTO_BOUNDARIES", "GRID_MAX_GRIDS",
        "DCA_DIP", "DCA_REBALANCE", "DCA_MAX_COUPLED", "RL_FEATURES", "RL_PARAMS", "RL_MAX_BATCH", "RL_MAX_MEMORY",
        "VP_MAX_BINS", "VP_NO_LABEL", "MM_NO_LABEL")]
    for prefix, codes in (("B200BT_PRIMARY_", {**_lib.PRIMARY, **_lib.PRIMARY_ADVANCED}),
                          ("B200BT_SEC_", {**_lib.SECONDARY, **_lib.SECONDARY_ADVANCED}),
                          ("B200BT_TRADE_MC_", _lib.TRADE_MC_METHODS), ("B200BT_MM_HAS_", _lib.MM_HAS),
                          ("B200BT_REGIME_", {n: i for i, n in enumerate(_lib.REGIMES)}),
                          ("B200BT_GRID_", {n: i for i, n in enumerate(_lib.GRID_TYPES)}),
                          ("B200BT_COL_", {n: i for i, n in enumerate(_lib.ANALYZER_COLUMNS)})):
        pairs += [(code, prefix + key.upper().removesuffix("_RATIO")) for key, code in codes.items()]
    return pairs


# macro families _lib mirrors whole: a macro of one of them that _lib lacks is drift too
COMPLETE_FAMILIES = ("B200BT_PRIMARY_", "B200BT_SEC_", "B200BT_TRADE_MC_", "B200BT_MM_HAS_", "B200BT_REGIME_",
                     "B200BT_EVENT_", "B200BT_COL_")


def _pointee_matches(argtype, ctype):
    if argtype is C.c_void_p:
        return True
    if not (isinstance(argtype, type) and issubclass(argtype, C._Pointer)) or ctype.pointers != 1:
        return False
    mirrors = [m for s, m in STRUCT_MIRRORS if s == ctype.base] if ctype.base.startswith("b200bt_") else [CTYPES[ctype.base]]
    return argtype._type_ in mirrors


def _matches(argtype, ctype):
    if ctype.pointers == 0:
        return argtype is CTYPES[ctype.base]
    if ctype == abi_header.CType("char", 1):
        return argtype in (C.c_char_p, C.c_void_p)
    return _pointee_matches(argtype, ctype)


def test_every_prototype_has_a_signature_and_every_signature_a_prototype():
    assert sorted(HEADER.prototypes) == _lib.exported_symbols()


@pytest.mark.parametrize("name", sorted(HEADER.prototypes))
def test_signature_matches_prototype(name):
    ret, params = HEADER.prototypes[name]
    res, args = _lib._SIGNATURES[name]
    assert _matches(res, ret), f"{name} returns {ret}, bound as {res}"
    assert len(args) == len(params), f"{name} takes {len(params)} arguments, bound with {len(args)}"
    for i, (argtype, ctype) in enumerate(zip(args, params)):
        assert _matches(argtype, ctype), f"{name} argument {i} is {ctype}, bound as {argtype}"


def _mirror_layout(mirror):
    """[(name, numpy base dtype, dims, offset, size)] and the total size of a Structure or a row dtype."""
    if isinstance(mirror, type) and issubclass(mirror, C.Structure):
        rows = []
        for name, t in mirror._fields_:
            dims = []
            while issubclass(t, C.Array):
                dims.append(t._length_)
                t = t._type_
            f = getattr(mirror, name)
            rows.append((name, np.dtype(t), tuple(dims), f.offset, f.size))
        return rows, C.sizeof(mirror)
    dt = np.dtype(mirror)
    return [(n, dt.fields[n][0].base, dt.fields[n][0].shape, dt.fields[n][1], dt.fields[n][0].itemsize)
            for n in dt.names], dt.itemsize


@pytest.mark.parametrize("struct, mirror", STRUCT_MIRRORS, ids=[
    s + ("-names" if isinstance(m, tuple) else "-dtype" if not isinstance(m, type) else "") for s, m in STRUCT_MIRRORS])
def test_struct_mirror_matches_header(struct, mirror):
    s = HEADER.structs[struct]
    assert s.size == s.comment, f"{struct}: {s.size} bytes, its comment says {s.comment}"
    if isinstance(mirror, tuple):
        assert [(f.name, f.ctype, f.dims) for f in s.fields] == [
            (n, "uint64_t" if n == "trade_hash" else "double", ()) for n in mirror]
        return
    rows, size = _mirror_layout(mirror)
    want = [(f.name, np.dtype(CTYPES[f.ctype]), f.dims, f.offset, f.size) for f in s.fields]
    assert rows == want
    assert size == s.size


def test_every_header_struct_is_mirrored_or_built_without_a_mirror():
    assert set(HEADER.structs) == {s for s, _ in STRUCT_MIRRORS} | set(NO_HOST_MIRROR)
    for struct, names in NO_HOST_MIRROR.items():
        assert [(f.name, f.ctype, f.dims) for f in HEADER.structs[struct].fields] == [(n, "int32_t", ()) for n in names]


def test_mirrored_constants_match_header():
    pairs = _constants()
    assert {macro: value for value, macro in pairs} == {macro: HEADER.defines.get(macro) for _, macro in pairs}
    mirrored = {macro for _, macro in pairs}
    assert {m for m in HEADER.defines if m.startswith(COMPLETE_FAMILIES)} <= mirrored
