"""TensorBoard summaries and alignment plots without TensorFlow (dc_tts_b200/summary.py, utils.plot_alignment): event
files framed and checksummed as TFRecords, PNG images with TF 1.x's float normalisation, and the tag set and values of the
reference's own training graphs (refshim_summaries.npz, tests/golden/make_golden_refchecks_summaries.py) rebuilt from the
oracle's forward."""
import io
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch

from conftest import ROOT, golden
from dc_tts_b200 import summary
from dc_tts_b200.hyperparams import Hyperparams as hp
from dc_tts_b200.params import init_params
from oracle import ref_train as rtr

import ref_train_bucket as rtb

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_refchecks_summaries import SSRN_SEED, SSRN_T, T2M_SEED, t2m_batch      # noqa: E402
from make_golden_refchecks_bucket import ssrn_batch                                  # noqa: E402


def _decode_png(data, use_pil=True):
    """(H, W) or (H, W, 3) uint8 pixels of a PNG: PIL when it is installed, else a zlib decoder of unfiltered rows."""
    if use_pil:
        try:
            from PIL import Image
            return np.asarray(Image.open(io.BytesIO(data)))
        except ImportError:
            pass
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, hdr = 8, b"", None
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(kind + body) & 0xffffffff
        if kind == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"IDAT":
            idat += body
        pos += 12 + n
    w, h, depth, color = hdr[:4]
    ch = {0: 1, 2: 3}[color]
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + w * ch)
    assert depth == 8 and not raw[:, 0].any()
    px = raw[:, 1:]
    return px if ch == 1 else px.reshape(h, w, 3)


def _tf_normalised(x):
    """TF 1.x's image summary for float input, restated: min/max over finite pixels; min >= 0 -> x * 255 / max, else
    x * 127 / max|x| + 128 (scale 0 below 1e-6); truncated to uint8; non-finite pixels 255."""
    x = np.asarray(x, np.float32)
    fin = np.isfinite(x)
    lo, hi = (x[fin].min(), x[fin].max()) if fin.any() else (0.0, 0.0)
    if lo >= 0:
        scale, off = (0.0 if hi < 1e-6 else np.float32(255) / np.float32(hi)), 0.0
    else:
        m = max(-lo, abs(hi))
        scale, off = (0.0 if m < 1e-6 else np.float32(127) / np.float32(m)), 128.0
    out = np.zeros(x.shape, np.uint8)
    out[fin] = np.clip(np.trunc(x[fin] * np.float32(scale) + np.float32(off)), 0, 255).astype(np.uint8)
    out[~fin] = 255
    return out


def _image_cases():
    rng = np.random.default_rng(0)
    pos = rng.uniform(0, 1, (hp.n_mels, 53)).astype(np.float32)
    mixed = rng.normal(0, 2, (hp.n_mels, 53)).astype(np.float32)
    nan = pos.copy(); nan[3, 5] = np.nan; nan[7, 0] = np.inf
    return {"positive": pos, "mixed": mixed, "zero": np.zeros((hp.n_mels, 53), np.float32), "nan": nan}


@pytest.mark.parametrize("case", ["positive", "mixed", "zero", "nan"])
def test_image_summary_decodes_to_tf_normalisation(case):
    x = _image_cases()[case]
    vals = summary.parse_summary(summary.image("train/mel_gt", x[None]))
    assert [t for t, _ in vals] == ["train/mel_gt/image/0"]
    img = vals[0][1]
    assert (img["height"], img["width"], img["colorspace"]) == (hp.n_mels, 53, 1)
    for use_pil in (True, False):
        px = _decode_png(img["png"], use_pil)
        assert px.shape == (hp.n_mels, 53)
        assert np.array_equal(px, _tf_normalised(x))


def test_event_file_records_and_checksums(tmp_path):
    w = summary.FileWriter(str(tmp_path))
    for step in (1, 2, 7):
        w.add_summary(summary.merge(summary.scalar("train/loss_mels", 0.5 / step), summary.scalar("lr", 1e-3 * step)), step)
    w.flush(); w.close()
    assert os.path.basename(w.path).startswith("events.out.tfevents.")
    ev = summary.read_events(w.path)
    assert ev[0]["file_version"] == "brain.Event:2" and "summary" not in ev[0]
    assert [e["step"] for e in ev[1:]] == [1, 2, 7]
    for e, step in zip(ev[1:], (1, 2, 7)):
        vals = dict(e["summary"])
        assert vals["train/loss_mels"] == np.float32(0.5 / step) and vals["lr"] == np.float32(1e-3 * step)
        assert e["wall_time"] >= ev[0]["wall_time"]
    data = bytearray(open(w.path, "rb").read())
    data[-6] ^= 1                                                  # one flipped bit in the last record's payload
    open(w.path, "wb").write(bytes(data))
    with pytest.raises(ValueError, match="checksum"):
        summary.read_events(w.path)


def test_event_file_loads_in_tensorboard(tmp_path, monkeypatch):
    # tensorboard imports tensorflow when it can: hide the TF stand-in other tests install, so it takes its own stub
    monkeypatch.setitem(sys.modules, "tensorflow", None)
    loader = pytest.importorskip("tensorboard.backend.event_processing.event_file_loader")
    w = summary.FileWriter(str(tmp_path))
    for step in (3, 4):
        w.add_summary(summary.scalar("train/loss_att", 0.25 * step), step)
    w.close()
    events = list(loader.EventFileLoader(w.path).Load())
    assert events[0].file_version == "brain.Event:2"
    got = [(e.step, v.tag, v.simple_value if v.HasField("simple_value") else float(v.tensor.float_val[0]))
           for e in events[1:] for v in e.summary.value]
    assert got == [(3, "train/loss_att", np.float32(0.75)), (4, "train/loss_att", np.float32(1.0))]


def _check_against_fixture(prefix, merged):
    g = golden("refshim_summaries.npz")
    tags = [str(t) for t in g[prefix + "_tags"]]
    ours = summary.parse_summary(merged)
    image_tags = [t for i, t in enumerate(tags) if g["%s_value_%d" % (prefix, i)].ndim == 4]
    assert [t for t, _ in ours] == [t + "/image/0" if t in image_tags else t for t in tags]
    for i, (t, (_, v)) in enumerate(zip(tags, ours)):
        ref = g["%s_value_%d" % (prefix, i)]
        if ref.ndim == 4:                                          # (1, C, T, 1): the tensor the reference's image op sees
            px = _decode_png(v["png"]).astype(np.int32)
            assert px.shape == ref.shape[1:3], t
            x = ref[0, :, :, 0].astype(np.float64)
            want = _tf_normalised(x).astype(np.int32)
            # the network outputs agree to ~1e-6, not bit for bit: a pixel whose scaled value lies within 1e-3 of an
            # integer may truncate to the neighbouring level; every other pixel is the reference's exactly
            scaled = x * 255.0 / x.max() if x.min() >= 0 else x * 127.0 / np.abs(x).max() + 128.0
            edge = np.abs(scaled - np.round(scaled)) < 1e-3
            assert np.array_equal(px[~edge], want[~edge]), t
            assert np.abs(px[edge] - want[edge]).max(initial=0) <= 1 and edge.mean() < 0.01, (t, edge.mean())
        else:
            assert abs(v - float(ref)) <= 2e-6 * max(1.0, abs(float(ref))), (t, v, float(ref))
    return g


def test_text2mel_summaries_vs_reference_training_graph():
    """train.py:100-104,123 on the fixture's batch: the oracle forward plus summary.train_summary give the reference
    graph's tags in its order, its scalars to 2e-6 and its images pixel for pixel (mels[:1] and Y[:1], transposed)."""
    P = init_params(0, "perturbed")
    L, mels = t2m_batch()
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.text2mel_names()}
    with torch.no_grad():
        o = rtb.forward(W, L, mels, T2M_SEED, hp.dropout_rate)
    losses = {k: float(o[k]) for k in ("loss_mels", "loss_bd1", "loss_att")}
    g = _check_against_fixture("t2m", summary.train_summary(1, losses, mels, o["Y"].numpy(), rtr.learning_rate(0)))
    assert np.abs(o["Y"].numpy() - g["t2m_Y"]).max() < 2e-5
    assert np.abs(o["alignments"].numpy() - g["t2m_alignments"]).max() < 2e-5


def test_ssrn_summaries_vs_reference_training_graph():
    P = init_params(0, "perturbed")
    mels, mags = ssrn_batch(SSRN_T)
    W = {n: torch.tensor(np.asarray(P[n], np.float32)) for n in rtr.ssrn_names()}
    with torch.no_grad():
        o = rtr.forward_ssrn(W, mels, mags, SSRN_SEED)
    losses = {k: float(o[k]) for k in ("loss_mags", "loss_bd2")}
    g = _check_against_fixture("ssrn", summary.train_summary(2, losses, mags, o["Z"].numpy(), rtr.learning_rate(0)))
    assert np.abs(o["Z"].numpy() - g["ssrn_Z"]).max() < 2e-5


def test_plot_alignment_png(tmp_path):
    from dc_tts_b200.utils import _viridis, plot_alignment
    a = np.random.default_rng(1).uniform(0, 1, (37, 53)).astype(np.float32)
    path = plot_alignment(a, "001k", str(tmp_path / "logdir"))
    assert path == str(tmp_path / "logdir" / "alignment_001k.png")
    px = _decode_png(open(path, "rb").read())
    k = px.shape[0] // 37
    assert k >= 1 and px.shape == (37 * k, 53 * k, 3)
    cmap = _viridis()
    assert np.array_equal(px[0, 0], cmap[int(np.floor((a[0, 0] - a.min()) / (a.max() - a.min()) * 255 + 0.5))])
    i, j = np.unravel_index(np.argmax(a), a.shape)                 # row 0 at the top, T along the columns
    assert np.array_equal(px[i * k, j * k], cmap[255])
    i, j = np.unravel_index(np.argmin(a), a.shape)
    assert np.array_equal(px[i * k + k - 1, j * k + k - 1], cmap[0])
