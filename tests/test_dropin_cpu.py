"""CPU: how gsx.dropin installs the device readers and writers and falls back to the reference's methods.  The
install_reader / install_writer rules over every row of the format table, through stub decode and prepare functions;
the real prepare and decode functions on a stand-in class, which on a machine without a CUDA device fail at their first
device allocation and so must fall back; the refusals prepare makes before any device work; patch() with stub
gsconverter.formats modules; and patch()'s ValueErrors.  The accepting path, with the bytes it writes, is checked in the
GPU suites of each codec."""
import json
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = Path(__file__).resolve().parent / "golden"

KEYWORDS = ("sog", "codecs", "readers", "sog_reader", "ply", "sog_webp", "spz_gzip", "sog_reader_webp", "parquet")
HOST = dict.fromkeys(KEYWORDS, "host")
CLASSES = (("splat", "SplatFormat"), ("ksplat", "KSplatFormat"), ("spz", "SpzFormat"),
           ("compressed_ply", "CompressedPlyFormat"), ("sog", "SogFormat"), ("ply_3dgs", "Ply3DGSFormat"),
           ("ply_cc", "PlyCCFormat"), ("parquet", "ParquetFormat"))
SIDES = [(name, "read") for _, name in CLASSES if name != "ParquetFormat"] + [(name, "write") for _, name in CLASSES]
FLIP = {"host": "device", "device": "host", "3dgs": "cc", "cc": "3dgs"}


def table():
    """{(class, "read" / "write"): (gsx function, install options)} of dropin's format table, all keywords "host"."""
    from gsx import dropin
    out = {}
    for _, name, reader, writer in dropin._formats(HOST):
        for method, side in (("read", reader), ("write", writer)):
            if side is not None:
                out[(name, method)] = side[1:]
    return out


class StandIn:
    """A reference format class: records each call with the global RNG state it saw, returns "reference"."""

    def __init__(self):
        self.calls = []
        self.metadata = "untouched"
        self.extra_elements = "untouched"

    def read(self, path, *args, **kwargs):
        self.calls.append(("read", path, args, kwargs, np.random.get_state()))
        return "reference"

    def write(self, data, path, *args, **kwargs):
        self.calls.append(("write", data, path, args, kwargs, np.random.get_state()))
        return "reference"


def rng_equal(a, b) -> bool:
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def install(cls, method, fn, options):
    from gsx import dropin
    (dropin.install_reader if method == "read" else dropin.install_writer)(cls, fn, **options)


def test_table_has_every_class_and_direction(gsx_lib):
    from gsx import dropin
    assert [(m, n) for m, n, *_ in dropin._formats(HOST)] == list(CLASSES)
    assert sorted(table()) == sorted(SIDES)


@pytest.mark.parametrize("name, method", SIDES)
def test_wrapper_rules(name, method, gsx_lib, tmp_path):
    _, options = table()[(name, method)]
    seen, refuse = [], [True]

    class Dec:                                            # what a decode returns
        metadata = {"count": 1} if name == "KSplatFormat" else None

        def to_host(self):
            return "device"

    def decode(path, **opts):                             # draws from the RNG, then refuses or accepts
        np.random.random(5)
        seen.append(opts)
        if refuse[0]:
            raise ValueError("refused")
        return Dec()

    def prepare(self, data, *args, **kwargs):
        np.random.random(5)
        seen.append(dict(self._gsx_options["write"]))
        if refuse[0]:
            raise ValueError("refused")
        return lambda path: Path(path).write_bytes(b"device")

    stub = decode if method == "read" else prepare
    cls = type(f"{name}_{method}", (StandIn,), {})
    install(cls, method, stub, {**options, "probe": 1})
    install(cls, method, stub, {**options, "probe": 1})              # installing twice keeps the original
    assert getattr(cls, f"_gsx_reference_{method}") is getattr(StandIn, method)
    assert getattr(cls, method) is not getattr(StandIn, method)
    # refused: the original, with the same arguments and the RNG as it was on entry; nothing written to path
    obj, path = cls(), tmp_path / "out"
    np.random.seed(5)
    state = np.random.get_state()
    if method == "read":
        assert obj.read(str(path), 7, level=4) == "reference"
        assert obj.calls[0][:4] == ("read", str(path), (7,), {"level": 4})
        assert obj.metadata == "untouched" and obj.extra_elements == "untouched"
    else:
        data = np.zeros(3, [("x", "<f4")])
        assert obj.write(data, path, 7, level=4) == "reference"
        assert obj.calls[0][1] is data and obj.calls[0][2:5] == (path, (7,), {"level": 4})
        assert not path.exists()
    assert len(obj.calls) == 1 and rng_equal(obj.calls[0][-1], state)
    # a second install with new options: the wrapper stays, the new options are the ones used
    changed = {k: FLIP.get(v, v) for k, v in options.items() if k != "after"}
    wrapper = getattr(cls, method)
    install(cls, method, stub, {**options, **changed, "probe": 2})
    assert getattr(cls, method) is wrapper
    refuse[0] = False
    obj = cls()
    if method == "read":
        assert obj.read(str(path)) == "device" and obj.calls == []
        assert obj.metadata == (Dec.metadata if Dec.metadata is not None else "untouched")
        assert obj.extra_elements == ([] if "after" in options else "untouched")
    else:
        assert obj.write(np.zeros(3, [("x", "<f4")]), path) is None and obj.calls == []
        assert path.read_bytes() == b"device"
    plain = {k: v for k, v in options.items() if k != "after"}
    assert seen == [{**plain, "probe": 1}, {**changed, "probe": 2}]


def writer_input():
    from gsx import synth
    return synth.structured(300, "mixed")


def reader_input(name) -> bytes:
    """A file the reference reads, from the goldens."""
    if name == "SogFormat":
        return np.load(GOLDEN / "g14_reference_sog_reader_small.npz")["custom_names_file"].tobytes()
    if name in ("Ply3DGSFormat", "PlyCCFormat"):
        return np.load(GOLDEN / "g15_reference_ply_small.npz")["read_3dgs_extras_file"].tobytes()
    case = {"SplatFormat": "splat_writer_edge", "KSplatFormat": "ksplat_multisection", "SpzFormat": "spz_writer_edge",
            "CompressedPlyFormat": "cply_order"}[name]
    return np.load(GOLDEN / "g13_reference_readers_small.npz")[f"{case}_file"].tobytes()


@pytest.mark.parametrize("name, method", SIDES)
def test_real_codecs_fall_back_without_a_device(name, method, gsx_lib, tmp_path):
    """The real prepare and decode functions of each row, installed as patch() installs them: with no CUDA device they
    fail at their first device allocation, and the call reaches the original with its arguments, nothing written."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device takes the accepting path; the GPU suites check it")
    fn, options = table()[(name, method)]
    cls = type(f"{name}_{method}", (StandIn,), {})
    install(cls, method, fn, options)
    obj = cls()
    np.random.seed(3)
    state = np.random.get_state()
    if method == "read":
        src = tmp_path / "in"
        src.write_bytes(reader_input(name))
        assert obj.read(str(src), level=4) == "reference"
        assert obj.calls[0][:4] == ("read", str(src), (), {"level": 4})
    else:
        data, path = writer_input(), tmp_path / "out"
        assert obj.write(data, path, compression_level=1) == "reference"
        assert obj.calls[0][1] is data and obj.calls[0][2:5] == (path, (), {"compression_level": 1})
        assert not path.exists()
    assert len(obj.calls) == 1 and rng_equal(obj.calls[0][-1], state)


@pytest.mark.parametrize("name", ["SplatFormat", "SpzFormat", "CompressedPlyFormat", "SogFormat", "Ply3DGSFormat",
                                  "PlyCCFormat", "ParquetFormat"])
def test_prepare_refuses_positional_arguments(name, gsx_lib):
    """Their reference write takes (data, path, **kwargs): the positional argument goes on to the reference, which
    raises the TypeError.  KSplatFormat.write takes compression_level positionally, so it is not here."""
    prepare, _ = table()[(name, "write")]
    with pytest.raises(TypeError, match="positional arguments"):
        prepare(StandIn(), writer_input(), 2)


@pytest.mark.parametrize("name", ["Ply3DGSFormat", "PlyCCFormat"])
def test_ply_prepare_refuses_extra_elements(name, gsx_lib):
    prepare, _ = table()[(name, "write")]
    with pytest.raises(ValueError, match="extra_elements"):
        prepare(StandIn(), writer_input(), extra_elements=["camera"])


@pytest.mark.parametrize("name, what", [("CompressedPlyFormat", "compressed PLY"), ("SogFormat", "SOG")])
def test_prepare_refuses_records_that_are_not_packed_f32(name, what, gsx_lib):
    prepare, _ = table()[(name, "write")]
    b = np.zeros(10, dtype=[("x", "f4"), ("y", "f4"), ("z", "f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    with pytest.raises(ValueError, match=f"{what} on the device needs packed all-float32 records"):
        prepare(StandIn(), b)


PATCH_PROBE = textwrap.dedent("""
    import json, sys, types
    sys.path[:0] = [{root!r}, {pkg!r}]
    import gsconverter
    fm = types.ModuleType("gsconverter.formats"); fm.__path__ = []
    sys.modules["gsconverter.formats"] = fm
    classes = []
    for mod, name in {classes!r}:
        m = types.ModuleType("gsconverter.formats." + mod)
        cls = type(name, (), {{"read": lambda self, *a, **k: None, "write": lambda self, *a, **k: None}})
        setattr(m, name, cls)
        sys.modules[m.__name__] = m
        classes.append(cls)
    from gsx import dropin
    assert dropin.patch(require_cuda=False, {kw})
    print(json.dumps({{c.__name__ + "." + m: c.__dict__.get("_gsx_options", {{}}).get(m) for c in classes
                       for m in ("read", "write") if "_gsx_reference_" + m in c.__dict__}}))
""")

CPLY_WRITE = {"CompressedPlyFormat.write": {}}           # installed whatever the keywords
CODECS = {f"{c}.write": {} for c in ("SplatFormat", "KSplatFormat")}
READERS = {f"{c}.read": {} for c in ("SplatFormat", "KSplatFormat", "SpzFormat", "CompressedPlyFormat")}
PLY = {"Ply3DGSFormat.read": {"flavor": "3dgs"}, "Ply3DGSFormat.write": {"flavor": "3dgs"},
       "PlyCCFormat.read": {"flavor": "cc"}, "PlyCCFormat.write": {"flavor": "cc"}}


@pytest.mark.parametrize("kw, want", [
    ("", CPLY_WRITE),
    ("codecs='host'", CPLY_WRITE),
    ("codecs='device'", {**CPLY_WRITE, **CODECS, "SpzFormat.write": {"gzip": "host"}}),
    ("codecs='device', spz_gzip='device'", {**CPLY_WRITE, **CODECS, "SpzFormat.write": {"gzip": "device"}}),
    ("readers='host'", CPLY_WRITE),
    ("readers='device'", {**CPLY_WRITE, **READERS}),
    ("readers='device', codecs='device'", {**CPLY_WRITE, **READERS, **CODECS, "SpzFormat.write": {"gzip": "host"}}),
    ("sog_reader='host'", CPLY_WRITE),
    ("sog_reader='device'", {**CPLY_WRITE, "SogFormat.read": {"webp": "host"}}),
    ("sog_reader='device', sog='device'", {**CPLY_WRITE, "SogFormat.read": {"webp": "host"},
                                           "SogFormat.write": {"webp": "host"}}),
    ("sog='device', sog_webp='device', sog_reader='device', sog_reader_webp='device'",
     {**CPLY_WRITE, "SogFormat.read": {"webp": "device"}, "SogFormat.write": {"webp": "device"}}),
    ("ply='host'", CPLY_WRITE),
    ("ply='device'", {**CPLY_WRITE, **PLY}),
    ("parquet='host'", CPLY_WRITE),
    ("parquet='device'", {**CPLY_WRITE, "ParquetFormat.write": {}}),
])
def test_patch_installs_what_the_keywords_ask(kw, want, gsx_lib):
    """Which methods of the eight reference classes patch() replaces, and the options each is installed with."""
    src = PATCH_PROBE.format(root=str(ROOT), pkg=str(ROOT / "3dgsconverter_b200"), kw=kw, classes=CLASSES)
    out = subprocess.run([sys.executable, "-c", src], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert json.loads(out.stdout.strip().splitlines()[-1]) == want


@pytest.mark.parametrize("keyword", KEYWORDS)
@pytest.mark.parametrize("value", ["gpu", "cuda"])
def test_patch_refuses_unknown_values(keyword, value):
    from gsx import dropin
    with pytest.raises(ValueError, match=f"{keyword} must be 'host' or 'device'"):
        dropin.patch(require_cuda=False, **{keyword: value})


@pytest.mark.parametrize("kw", [
    dict(spz_gzip="device"), dict(codecs="host", spz_gzip="device"), dict(codecs="device", spz_gzip="cuda"),
    dict(codecs="device", spz_gzip="gpu"),
    dict(sog_webp="device"), dict(sog="device", sog_webp="cuda"), dict(sog="device", sog_webp="gpu"),
    dict(sog_reader_webp="device"), dict(sog_reader="device", sog_reader_webp="gpu"),
    dict(sog_reader="gpu"), dict(parquet="gpu"), dict(ply="gpu"),
])
def test_patch_refuses_invalid_values_and_dependencies(kw):
    """Every ValueError the per-format tests checked, raised before patch() touches anything, with or without
    require_cuda."""
    from gsx import dropin
    for require_cuda in (True, False):
        with pytest.raises(ValueError):
            dropin.patch(require_cuda=require_cuda, **kw)
