"""CPU tests of the JPEG decode: the numpy oracle bitwise against what Pillow decoded (tests/golden/jpeg.npz,
oracle/gen_golden_jpeg.py), the library's host plan (dimensions, scan and output offsets), every refused kind of stream refused
by name with nothing launched, and the dataset-side byte packing."""
import ctypes as C
import hashlib
import json
import os
import re
import struct

import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "jpeg.npz"))
CASES = json.loads(str(GOLDEN["cases"]))["cases"]


def jpg(name):
    return GOLDEN["jpg_" + name].tobytes()


def golden_ok(case, mode, px):
    if "sha256_" + mode in case:
        return hashlib.sha256(px.tobytes()).hexdigest() == case["sha256_" + mode]
    ref = GOLDEN["px_%s_%s" % (mode, case["name"])]
    return px.shape == ref.shape and px.tobytes() == ref.tobytes()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_oracle_matches_pillow(case):
    for mode in ("RGB", "L"):
        px, status = J.decode(jpg(case["name"]), mode, with_status=True)
        assert status == J.OK
        assert px.shape == (case["height"], case["width"], 3 if mode == "RGB" else 1)
        assert golden_ok(case, mode, px), mode


def test_golden_covers_the_issue_matrix():
    names = [c["name"] for c in CASES]
    for size in ("1x1", "7x9", "8x8", "15x17", "16x16", "37x23", "341x255", "340x256", "480x360"):
        assert any(n.startswith(size + "_") for n in names), size
    for q in (5, 50, 75, 90, 95, 100):
        assert any(c["encoder"].get("quality") == q for c in CASES), q
    for key in ("optimize", "restart_marker_blocks", "restart_marker_rows"):
        assert any(key in c["encoder"] for c in CASES), key
    assert {c["subsampling"] for c in CASES} == {"444", "422", "420", "gray"}
    assert {"flat", "saturated", "checker", "noise", "smooth"} <= {c["content"] for c in CASES}
    assert os.path.getsize(os.path.join(ROOT, "tests", "golden", "jpeg.npz")) < 1_100_000


def test_restart_intervals_are_split_where_the_markers_are():
    hdr = J.parse(jpg("37x23_420_smooth_rst_blocks"))
    ivs, _ = J._intervals(jpg("37x23_420_smooth_rst_blocks"), hdr["scan"])
    mcux, mcuy, _ = J.geometry(hdr)
    assert hdr["restart"] >= 1 and len(ivs) == -(-(mcux * mcuy) // hdr["restart"])
    assert [k for k, _ in ivs[1:]] == [i % 8 for i in range(len(ivs) - 1)]


# ---- the library's host plan ----------------------------------------------------------------------------------------------------
def _plan(blobs, channels=3):
    from ops.jpeg import JpegPlan
    ends = np.cumsum([len(b) for b in blobs])
    buf = np.frombuffer(b"".join(blobs), np.uint8)
    ch = [channels] * len(blobs) if isinstance(channels, int) else channels
    return JpegPlan(buf, ends - [len(b) for b in blobs], ends, ch), ends - [len(b) for b in blobs]


def test_host_plan_dimensions_and_offsets():
    names = [c["name"] for c in CASES]
    blobs = [jpg(n) for n in names]
    ch = [3 if i % 3 else 1 for i in range(len(blobs))]
    plan, starts = _plan(blobs, ch)
    out = 0
    for i, (n, b) in enumerate(zip(names, blobs)):
        hdr, im = J.parse(b), plan.images[i]
        mcux, mcuy, _ = J.geometry(hdr)
        assert (im.width, im.height, im.components, im.channels) == (hdr["width"], hdr["height"], len(hdr["comps"]), ch[i]), n
        assert (im.h_samp, im.v_samp) == ((hdr["comps"][0][1], hdr["comps"][0][2]) if len(hdr["comps"]) == 3 else (1, 1)), n
        assert im.scan_offset == starts[i] + hdr["scan"], n
        _, end = J._intervals(b, hdr["scan"])
        assert im.scan_bytes == end - hdr["scan"], n
        assert im.restart_interval == hdr["restart"]
        assert im.intervals == -(-(mcux * mcuy) // (hdr["restart"] or mcux * mcuy)), n
        assert im.out_offset == out, n
        out += im.width * im.height * ch[i]
    assert plan.out_bytes == out
    assert plan.table_bytes % 256 == 0
    # identical Huffman / quantisation tables are stored once: 122 images of a few table sets stay small
    assert plan.table_bytes < 400_000


def _segments(b):
    """[(marker, start, end)] of the header segments of b up to SOS (start: the marker's 0xFF)"""
    out, p = [], 2
    while True:
        m = b[p + 1]
        L = struct.unpack(">H", b[p + 2:p + 4])[0]
        out.append((m, p, p + 2 + L))
        if m == 0xDA:
            return out
        p += 2 + L


def _patch(b, marker, rel, value):
    """b with byte `rel` of the first `marker` segment's payload (after the length) set to value"""
    m, s, e = next(x for x in _segments(b) if x[0] == marker)
    b = bytearray(b)
    b[s + 4 + rel] = value
    return bytes(b)


def _without_app0(b):
    m, s, e = next(x for x in _segments(b) if x[0] == 0xE0)
    return b[:s] + b[e:]


def _with_marker(b, old, new):
    s = next(s for k, s, e in _segments(b) if k == old)
    return b[:s + 1] + bytes([new]) + b[s + 2:]


def _refused():
    b444 = next(jpg(c["name"]) for c in CASES if c["subsampling"] == "444" and c["width"] == 16)
    b420 = next(jpg(c["name"]) for c in CASES if c["subsampling"] == "420" and c["width"] == 16)
    sof = lambda b, m: _with_marker(b, 0xC0, m)
    nf4 = b"\xff\xd8\xff\xc0\x00\x14\x08\x00\x10\x00\x10\x04" + b"".join(bytes([i, 0x11, 0]) for i in (1, 2, 3, 4)) + b"\xff\xd9"
    adobe = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"          # APP14, transform 0
    no_jfif = _without_app0(b444)
    sof_s = next(s for k, s, e in _segments(no_jfif) if k == 0xC0)
    sos_s = next(s for k, s, e in _segments(no_jfif) if k == 0xDA)
    rgb_ids = bytearray(no_jfif)
    for j, cid in enumerate((82, 71, 66)):
        rgb_ids[sof_s + 4 + 6 + 3 * j] = cid
        rgb_ids[sos_s + 4 + 1 + 2 * j] = cid
    sos420 = next(s for k, s, e in _segments(b420) if k == 0xDA)
    dht_s, dht_e = next((s, e) for k, s, e in _segments(b420) if k == 0xC4)
    return [
        ("progressive", GOLDEN["jpg_progressive"].tobytes(), 4, "progressive JPEG (SOF2) is not supported"),
        ("lossless", sof(b420, 0xC3), 4, "lossless JPEG (SOF3) is not supported"),
        ("hierarchical", sof(b420, 0xC5), 4, "hierarchical JPEG (SOF5) is not supported"),
        ("arithmetic", sof(b420, 0xC9), 4, "arithmetic-coded JPEG (SOF9) is not supported"),
        ("12-bit", _patch(b420, 0xC0, 0, 12), 4, "12-bit samples are not supported"),
        ("cmyk", nf4, 4, "CMYK / YCCK JPEG is not supported"),
        ("adobe-rgb", no_jfif[:2] + adobe + no_jfif[2:], 4, "Adobe RGB (transform 0) JPEG is not supported"),
        ("rgb-ids", bytes(rgb_ids), 4, "RGB (component ids R, G, B) JPEG is not supported"),
        ("sampling-1x2", _patch(b420, 0xC0, 7, 0x12), 4, "sampling factors 12x11x11 are not supported"),
        ("sampling-chroma", _patch(b420, 0xC0, 10, 0x21), 4, "sampling factors 22x21x11 are not supported"),
        ("undefined-dc", bytes(bytearray(b420[:sos420 + 4 + 4]) + bytes([0x31]) + b420[sos420 + 4 + 5:]), 1,
         "scan references undefined DC Huffman table 3"),
        ("undefined-quant", _patch(b420, 0xC0, 8, 3), 1, "scan references undefined quantisation table 3"),
        ("truncated-header", b420[:(dht_s + dht_e) // 2], 1, "truncated header"),
        ("no-sos", b420[:sos420], 1, "truncated header (no SOS marker)"),
        ("not-jpeg", b"GIF89a\x00\x00", 1, "not a JPEG stream (no SOI marker)"),
    ]


REFUSED = _refused()


@pytest.mark.parametrize("kind, data, code, reason", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_streams_name_the_image_and_launch_nothing(kind, data, code, reason):
    from ops.jpeg import JpegRefused, decode_jpeg
    from ssn_b200._lib import lib
    with pytest.raises(J.JpegError, match=re.escape(reason)):
        J.parse(data)
    good = jpg(CASES[0]["name"])
    n0 = lib.ssnb_global_launch_count()
    with pytest.raises(JpegRefused) as e:
        _plan([good, good, data])
    assert e.value.image == 2 and e.value.reason == reason and e.value.code == code
    assert (lib.ssnb_last_error(None) or b"").decode() == "jpeg: image 2: " + reason
    # decode_jpeg refuses on the host, before it looks for a device
    with pytest.raises(ValueError, match=r"decode_jpeg: image 2 \(group 1, image 0\): " + re.escape(reason)):
        decode_jpeg([[good, good], [data, good]])
    assert lib.ssnb_global_launch_count() == n0


def test_decode_argument_checks_launch_nothing():
    from ssn_b200._lib import lib
    plan, _ = _plan([jpg(CASES[5]["name"])])
    n0 = lib.ssnb_global_launch_count()
    fake = 1 << 40           # never dereferenced: every check fails before a launch
    args = dict(table=fake, src=fake, src_bytes=plan.buf.size, out=fake, out_bytes=plan.out_bytes, status=fake, ws=fake,
                ws_bytes=plan.workspace_bytes)
    for bad in (dict(table=0), dict(out_bytes=plan.out_bytes - 1), dict(ws_bytes=plan.workspace_bytes - 1), dict(src_bytes=plan.buf.size - 1),
                dict(ws=fake + 16), dict(status=0)):
        a = dict(args, **bad)
        rc = lib.ssnb_jpeg_decode(plan.handle, a["table"], a["src"], a["src_bytes"], a["out"], a["out_bytes"], a["status"], a["ws"],
                                  a["ws_bytes"], None)
        assert rc == 1, bad
        assert (lib.ssnb_last_error(None) or b"").decode().startswith("jpeg_decode: ")
    assert lib.ssnb_jpeg_decode(None, fake, fake, 0, fake, 0, fake, fake, 0, None) == 1
    assert lib.ssnb_global_launch_count() == n0


def test_struct_layout():
    from ssn_b200._lib import JpegInput, JpegImageInfo
    assert C.sizeof(JpegInput) == 24 and C.sizeof(JpegImageInfo) == 56
    assert JpegImageInfo.scan_offset.offset == 32 and JpegImageInfo.out_offset.offset == 48


# ---- the dataset side -----------------------------------------------------------------------------------------------------------
def test_packed_groups_round_trip_and_concatenate():
    from ops.jpeg import pack_jpeg_group, unpack_jpeg_group, GroupToJpegBytes
    blobs = [jpg(c["name"]) for c in CASES[:5]]
    a, b = pack_jpeg_group(blobs[:2]), GroupToJpegBytes()(blobs[2:])
    assert a.dtype == torch.uint8 and a.dim() == 1
    buf, starts, ends = unpack_jpeg_group(torch.cat([a, b]))          # a video's proposals, as get_training_data cats them
    assert [buf[s:e].tobytes() for s, e in zip(starts, ends)] == blobs
    with pytest.raises(ValueError):
        unpack_jpeg_group(a[:-1])


def test_bytes_loader_keeps_the_reference_order(tmp_path):
    from ops.jpeg import JpegBytesLoader, GroupToJpegBytes, collate_jpeg, unpack_jpeg_group
    for k, name in enumerate(("img_00003.jpg", "x_00003.jpg", "y_00003.jpg")):
        (tmp_path / name).write_bytes(jpg(CASES[k]["name"]))

    class Data(JpegBytesLoader):          # the attributes SSNDataSet / BinaryDataSet's _load_image reads
        def __init__(self, modality, tmpl):
            self.modality, self.image_tmpl = modality, tmpl

    assert Data("RGB", "img_{:05d}.jpg")._load_image(str(tmp_path), 3) == [jpg(CASES[0]["name"])]
    assert Data("RGBDiff", "img_{:05d}.jpg")._load_image(str(tmp_path), 3) == [jpg(CASES[0]["name"])]
    flow = Data("Flow", "{}_{:05d}.jpg")._load_image(str(tmp_path), 3)
    assert flow == [jpg(CASES[1]["name"]), jpg(CASES[2]["name"])]
    samples = [(GroupToJpegBytes()(flow * (v + 1)), torch.tensor([v]), 0.5 * v) for v in range(2)]
    frames, labels, w = collate_jpeg(samples)
    assert isinstance(frames, list) and len(frames) == 2 and labels.tolist() == [[0], [1]] and w.tolist() == [0.0, 0.5]
    buf, s, e = unpack_jpeg_group(frames[1])
    assert [buf[a:b].tobytes() for a, b in zip(s, e)] == flow * 2


def test_model_frame_transforms_gain_a_decode_entry():
    import ssn_models
    for modality, mode in (("RGB", "RGB"), ("Flow", "L")):
        tf = ssn_models.SSN(4, 2, 5, 2, modality, base_model="BNInception", dropout=0).frame_transforms()
        assert tf.decode.keywords == {"mode": mode}
        assert {"sample_train_params", "train", "oversample", "center_crop", "to_uint8", "decode"} == set(vars(tf))
