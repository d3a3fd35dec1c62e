"""CPU: model files (fsn_model_file_write / fsn_model_file_config, model.save_model_file, fsnplus_b200.tools.export; DESIGN.md §3.15).

Round trips for six configurations, an independent numpy reader of the format as include/fsnplus_b200.h states it, the exporter on a
checkpoint, and every rejection with its message: bad magic or version, truncation at every item boundary and inside every item,
flipped bytes, trailing bytes, bad key lengths, unknown and missing config fields, a missing / extra / duplicate / mis-sized key, a
configuration fsn_model_create refuses, and writes that fail without leaving a file behind.  No compute calls."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ["model_kind", "num_freqs", "look_ahead", "sb_num_neighbors", "fb_num_neighbors", "fb_hidden", "sb_hidden", "num_layers",
          "output_size", "fb_act", "sb_act", "norm_type", "kersize[0]", "kersize[1]", "kersize[2]", "lstm_impl", "fast_math",
          "channel_attention", "rnn_type", "subband_num", "tcn_causal", "sb_tcn"]

# configuration name -> (model class, constructor keywords over the reference defaults)
CASES = {
    "plus_default": ("FullSubNet_Plus", {}),
    "sb_tcn": ("FullSubNet_Plus", dict(sequence_model="TCN")),
    "causal_tcn": ("FullSubNet_Plus", dict(causal_tcn=True)),
    "eca_sub2": ("FullSubNet_Plus", dict(channel_attention_model="ECA", subband_num=2)),
    "fsn_gru_cumulative": ("Model", dict(sequence_model="GRU", norm_type="cumulative_laplace_norm")),
    "wide": ("FullSubNet_Plus", dict(fb_num_neighbors=15)),
}


def case(name, seed=0, **over):
    """(model class name, constructor keywords, seeded state_dict as numpy arrays) of configuration `name`; `over` changes keywords."""
    cls, kw = CASES[name]
    if cls == "Model":
        cfg = dict(O.default_fsn_config(), **kw, **over)
        return cls, cfg, O.make_params_fsn(cfg, seed=seed)
    cfg = dict(O.default_plus_config(), **kw, **over)
    return cls, cfg, (S.make_params(cfg, seed=seed) if cfg["sequence_model"] == "TCN" else O.make_params_plus(cfg, seed=seed))


def build(name, seed=0, **over):
    """The Python module of configuration `name` with seeded parameters, in eval mode on the CPU."""
    from fsnplus_b200 import model as M
    cls, cfg, params = case(name, seed, **over)
    m = getattr(M, cls)(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    return m.eval()


def small():
    """A small fullsubnet.Model (F = 33, hidden 32): the base of the crafted files below."""
    return build("fsn_gru_cumulative", seed=3, num_freqs=33, sb_num_neighbors=3, fb_model_hidden_size=32, sb_model_hidden_size=32)


# ---- an independent implementation of the format -------------------------------------------------------------------------------

def file_hash(b):
    """The checksum: FNV-1a basis, then per 8-byte little-endian word (the last one zero-padded) h = (h ^ w) * prime, h ^= h >> 29."""
    b = bytes(b) + b"\0" * (-len(b) % 8)
    h, mask = 0xcbf29ce484222325, (1 << 64) - 1
    for w in np.frombuffer(b, "<u8").tolist():
        h = ((h ^ w) * 0x100000001b3) & mask
        h ^= h >> 29
    return h


def parse(b, verify_hash=True):
    """The file's parts: {"version", "fields": [(name, value)], "params": [(key, float32 array)], "items": [(offset, what)]} -- items
    lists where every item of the file starts, in order."""
    pos, items = 0, []

    def take(n, what):
        nonlocal pos
        items.append((pos, what))
        assert pos + n <= len(b), f"truncated at {what}"
        pos += n
        return b[pos - n:pos]
    assert take(8, "magic") == b"FSNMODEL"
    version, = struct.unpack("<I", take(4, "version"))
    nf, = struct.unpack("<I", take(4, "field count"))
    fields = []
    for _ in range(nf):
        ln, = struct.unpack("<H", take(2, "name length"))
        name = take(ln, "name").decode()
        fields.append((name, struct.unpack("<i", take(4, "value"))[0]))
    npar, = struct.unpack("<I", take(4, "parameter count"))
    params = []
    for _ in range(npar):
        ln, = struct.unpack("<H", take(2, "key length"))
        key = take(ln, "key").decode()
        numel, = struct.unpack("<q", take(8, "numel"))
        params.append((key, np.frombuffer(take(4 * numel, "data"), "<f4")))
    end = pos
    stored, = struct.unpack("<Q", take(8, "checksum"))
    assert pos == len(b), "trailing bytes"
    if verify_hash:
        assert stored == file_hash(b[:end])
    return dict(version=version, fields=fields, params=params, items=items)


def pack(fields, params, version=1, magic=b"FSNMODEL"):
    """A model file of these (name, value) fields and (key, array) records, with its checksum."""
    out = [magic, struct.pack("<II", version, len(fields))]
    for name, v in fields:
        out.append(struct.pack("<H", len(name)) + name.encode() + struct.pack("<i", v))
    out.append(struct.pack("<I", len(params)))
    for key, a in params:
        a = np.ascontiguousarray(a, "<f4").ravel()
        out.append(struct.pack("<H", len(key)) + key.encode() + struct.pack("<q", a.size) + a.tobytes())
    b = b"".join(out)
    return b + struct.pack("<Q", file_hash(b))


def cfg_fields(cfg):
    return [(n, cfg.kersize[int(n[-2])] if n.startswith("kersize") else getattr(cfg, n)) for n in FIELDS]


# ---- helpers around the C ABI ---------------------------------------------------------------------------------------------------

def file_config(lib, path):
    """(rc, message, config) of fsn_model_file_config."""
    from fsnplus_b200 import _lib
    cfg = _lib.FsnConfig()
    rc = lib.fsn_model_file_config(os.fsencode(path), C.byref(cfg))
    return rc, lib.fsn_last_error().decode(), cfg


def write(lib, path, cfg, params):
    """(rc, message) of fsn_model_file_write with (key, array) records."""
    from fsnplus_b200 import _lib
    arrs = [np.ascontiguousarray(a, np.float32).ravel() for _, a in params]
    n = len(params)
    keys = (C.c_char_p * n)(*[k.encode() for k, _ in params])
    data = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    numel = (C.c_int64 * n)(*[a.size for a in arrs])
    rc = lib.fsn_model_file_write(os.fsencode(path), C.byref(cfg), n, keys, data, numel)
    return rc, lib.fsn_last_error().decode()


def create_message(lib, cfg):
    """fsn_model_create's code and message for a configuration it refuses (it checks before it looks for a device)."""
    h = C.c_void_p()
    rc = lib.fsn_model_create(C.byref(cfg), C.byref(h))
    assert rc != 0
    return rc, lib.fsn_last_error().decode()


# ---- round trips ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASES))
def test_round_trip(built_lib, tmp_path, name):
    """save_model_file -> fsn_model_file_config returns every field; the numpy reader finds the format the header states: version 1,
    every fsn_config field by name in declaration order, exactly the state_dict's keys with their float32 values, and the checksum."""
    m = build(name)
    path = tmp_path / "m.fsn"
    m.save_model_file(path)
    rc, msg, cfg = file_config(built_lib, path)
    assert rc == 0, msg
    assert bytes(cfg) == bytes(m._cfg)
    b = path.read_bytes()
    f = parse(b, verify_hash=len(b) < (8 << 20))                       # the pure-Python hash of a large file takes long
    assert f["version"] == 1 and f["fields"] == cfg_fields(m._cfg)
    sd = m.state_dict()
    assert sorted(k for k, _ in f["params"]) == sorted(sd)
    for k, a in f["params"]:
        assert np.array_equal(a, sd[k].numpy().ravel()), k
    assert not os.path.exists(str(path) + ".tmp")


def test_checksum_of_a_small_file(built_lib, tmp_path):
    """The numpy reader's checksum on a small file, and a file packed by the numpy writer reads back in the library."""
    m = small()
    m.save_model_file(tmp_path / "a.fsn")
    b = (tmp_path / "a.fsn").read_bytes()
    f = parse(b)
    (tmp_path / "b.fsn").write_bytes(pack(f["fields"], f["params"]))
    assert (tmp_path / "b.fsn").read_bytes() == b
    rc, msg, cfg = file_config(built_lib, tmp_path / "b.fsn")
    assert rc == 0 and bytes(cfg) == bytes(m._cfg), msg


def test_written_in_spec_order(built_lib, tmp_path):
    """The records follow the configuration's key order whatever order the caller passes them in: the same weights give the same
    bytes."""
    from fsnplus_b200 import _lib
    m = small()
    sd = {k: m._host_param(v) for k, v in m.state_dict().items()}
    _lib.write_model_file(tmp_path / "a.fsn", m._cfg, sd)
    _lib.write_model_file(tmp_path / "b.fsn", m._cfg, dict(reversed(list(sd.items()))))
    assert (tmp_path / "a.fsn").read_bytes() == (tmp_path / "b.fsn").read_bytes()


def test_exporter(built_lib, tmp_path, capsys):
    """python -m fsnplus_b200.tools.export on a checkpoint saved from the CPU module built from the reference's inference.toml: the file's
    configuration is the module's, its records are the checkpoint's tensors, and the tool prints the file's size and key count."""
    from fsnplus_b200.tools import export, inference as T
    toml = tmp_path / "inference.toml"
    toml.write_text(open(os.path.join(ROOT, "tests", "golden", "inference_reference.toml")).read())
    conf = T.load_toml(toml)
    from fsnplus_b200 import model as M
    net = getattr(M, T.MODEL_PATHS[conf["model"]["path"]])(**conf["model"]["args"])
    params = O.make_params_plus(O.default_plus_config(), seed=4)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    torch.save({"model": net.state_dict(), "epoch": 7}, tmp_path / "ckpt.tar")
    out = tmp_path / "model.fsn"
    export.main(["-C", str(toml), "-M", str(tmp_path / "ckpt.tar"), "-O", str(out)])
    printed = capsys.readouterr().out
    assert f"{out.stat().st_size} bytes" in printed and f"{len(params)} parameters" in printed and "epoch 7" in printed, printed
    rc, msg, cfg = file_config(built_lib, out)
    assert rc == 0 and bytes(cfg) == bytes(net._cfg), msg
    f = parse(out.read_bytes(), verify_hash=False)
    assert len(f["params"]) == len(params)
    for k, a in f["params"]:
        assert np.array_equal(a, params[k].ravel()), k


# ---- rejections -----------------------------------------------------------------------------------------------------------------

@pytest.fixture
def small_file(built_lib, tmp_path):
    m = small()
    m.save_model_file(tmp_path / "ok.fsn")
    b = (tmp_path / "ok.fsn").read_bytes()
    return m, b, parse(b)


def _refused(lib, tmp_path, b, *needles):
    p = tmp_path / "bad.fsn"
    p.write_bytes(b)
    rc, msg, _ = file_config(lib, p)
    assert rc == -1, (rc, msg)
    for s in needles:
        assert s in msg, (s, msg)
    return msg


def test_bad_magic_and_version(built_lib, tmp_path, small_file):
    m, b, f = small_file
    _refused(built_lib, tmp_path, b"FSNMODEX" + b[8:], "bad magic")
    _refused(built_lib, tmp_path, pack(f["fields"], f["params"], version=2), "format version 2, this library reads version 1")
    _refused(built_lib, tmp_path, pack(f["fields"], f["params"], version=0), "format version 0")


def test_truncation_everywhere(built_lib, tmp_path, small_file):
    """A file cut at every item boundary, and one byte into every item, is refused naming the item's byte offset."""
    m, b, f = small_file
    for off, what in f["items"]:
        for cut in (off, off + 1):
            if cut >= len(b) or (cut == off + 1 and b[off:off + 1] == b""):
                continue
            msg = _refused(built_lib, tmp_path, b[:cut], "truncated", f"at byte {off} ")
            assert f"the file ends at byte {cut}" in msg, (what, cut, msg)


def test_flipped_bytes(built_lib, tmp_path, small_file):
    """One flipped byte in each section: the magic and the version are named, anything else fails the checksum."""
    m, b, f = small_file
    items = f["items"]
    first = {what: off for off, what in reversed(items)}
    flip = lambda i: b[:i] + bytes([b[i] ^ 0xFF]) + b[i + 1:]
    _refused(built_lib, tmp_path, flip(3), "bad magic")
    _refused(built_lib, tmp_path, flip(8), "format version 254")
    for where in (first["name"], first["value"], first["key"], first["data"] + 5, len(b) - 1):
        _refused(built_lib, tmp_path, flip(where), "checksum mismatch")


def test_trailing_bytes_and_key_lengths(built_lib, tmp_path, small_file):
    m, b, f = small_file
    _refused(built_lib, tmp_path, b + b"\0", "1 trailing bytes")
    for bad in ("", "k" * 256):
        params = [(bad, f["params"][0][1])] + f["params"][1:]
        _refused(built_lib, tmp_path, pack(f["fields"], params), f"key length {len(bad)}", "1..255")


def test_config_fields(built_lib, tmp_path, small_file):
    """An unknown field name is refused; a field the file does not name takes 0 (here sb_tcn, which older files lack)."""
    m, b, f = small_file
    _refused(built_lib, tmp_path, pack(f["fields"] + [("future_knob", 1)], f["params"]), 'unknown config field "future_knob"')
    _refused(built_lib, tmp_path, pack(f["fields"] + [("num_freqs", 33)], f["params"]), "config field num_freqs appears twice")
    p = tmp_path / "old.fsn"
    p.write_bytes(pack([x for x in f["fields"] if x[0] != "sb_tcn"], f["params"]))
    rc, msg, cfg = file_config(built_lib, p)
    assert rc == 0, msg
    assert cfg.sb_tcn == 0 and bytes(cfg) == bytes(m._cfg)


def test_key_set(built_lib, tmp_path, small_file):
    """A missing, extra, duplicate or mis-sized key is refused by the reader and by the writer, with the messages of
    fsn_model_finalize and fsn_model_set_param."""
    m, b, f = small_file
    params = f["params"]
    k0, a0 = params[0]
    cases = [(params[1:], f"missing parameter {k0}"), (params + [("sb_model.extra", a0)], "unexpected key sb_model.extra"),
             (params + [params[0]], f"duplicate key {k0}"),
             ([(k0, a0[:-1])] + params[1:], f"size mismatch for {k0}: expected {a0.size}, got {a0.size - 1}")]
    for recs, needle in cases:
        _refused(built_lib, tmp_path, pack(f["fields"], recs), needle)
        rc, msg = write(built_lib, tmp_path / "w.fsn", m._cfg, recs)
        assert rc == -1 and needle in msg, (needle, rc, msg)
        assert not (tmp_path / "w.fsn").exists()


def test_config_refused_like_create(built_lib, tmp_path, small_file):
    """A configuration fsn_model_create refuses gets create's code and message from the writer and from the reader."""
    from fsnplus_b200 import _lib
    m, b, f = small_file
    for field, v in (("num_layers", 5), ("model_kind", 7), ("sb_hidden", 100), ("norm_type", 9), ("sb_tcn", 1)):
        cfg = _lib.FsnConfig.from_buffer_copy(m._cfg)
        setattr(cfg, field, v)
        want = create_message(built_lib, cfg)
        assert write(built_lib, tmp_path / "w.fsn", cfg, f["params"]) == want
        assert not (tmp_path / "w.fsn").exists()
        fields = [(n, v if n == field else x) for n, x in f["fields"]]
        p = tmp_path / "bad.fsn"
        p.write_bytes(pack(fields, f["params"]))
        assert file_config(built_lib, p)[:2] == want


def test_failed_writes_leave_no_file(built_lib, tmp_path, small_file):
    """A directory that does not exist, a path that is a directory (the rename fails) and, for an ordinary user, a read-only directory:
    FSN_EINVAL naming the cause, and neither the file nor its temporary is left behind."""
    m, b, f = small_file
    rc, msg = write(built_lib, tmp_path / "missing" / "m.fsn", m._cfg, f["params"])
    assert rc == -1 and "cannot create" in msg and "No such file" in msg, msg
    assert not (tmp_path / "missing").exists()
    (tmp_path / "d.fsn").mkdir()
    rc, msg = write(built_lib, tmp_path / "d.fsn", m._cfg, f["params"])
    assert rc == -1 and "cannot rename" in msg, msg
    assert (tmp_path / "d.fsn").is_dir() and not (tmp_path / "d.fsn.tmp").exists()
    if os.geteuid() != 0:                                              # root writes into a read-only directory
        ro = tmp_path / "ro"
        ro.mkdir()
        ro.chmod(0o500)
        try:
            rc, msg = write(built_lib, ro / "m.fsn", m._cfg, f["params"])
            assert rc == -1 and "cannot create" in msg, msg
            assert os.listdir(ro) == []
        finally:
            ro.chmod(0o700)
    with pytest.raises(Exception, match="cannot create"):
        m.save_model_file(tmp_path / "missing" / "m.fsn")


def test_null_arguments(built_lib, tmp_path, small_file):
    m, b, f = small_file
    from fsnplus_b200 import _lib
    assert built_lib.fsn_model_file_config(None, C.byref(_lib.FsnConfig())) == -1
    assert built_lib.fsn_model_file_config(b"x", None) == -1
    assert built_lib.fsn_model_load(b"x", None) == -1
    assert built_lib.fsn_model_file_write(None, C.byref(m._cfg), 0, None, None, None) == -1
    assert built_lib.fsn_model_file_write(b"x", C.byref(m._cfg), -1, None, None, None) == -1
    assert b"negative" in built_lib.fsn_last_error()
    rc, msg, _ = file_config(built_lib, tmp_path / "none.fsn")
    assert rc == -1 and "cannot open" in msg
