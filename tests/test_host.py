"""CPU tests of the host side: text adaptor, config surface, C-ABI export table."""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from dc_tts_b200 import _lib, arch
from dc_tts_b200.data_load import load_data, load_vocab, text_normalize
from dc_tts_b200.hyperparams import Hyperparams as hp


def test_hyperparams_surface():
    # every attribute of the reference class (hyperparams.py:7-47) with its value
    want = dict(prepro=True, sr=22050, n_fft=2048, frame_shift=0.0125, frame_length=0.05, hop_length=275,
                win_length=1102, n_mels=80, power=1.5, n_iter=50, preemphasis=.97, max_db=100, ref_db=20,
                r=4, dropout_rate=0.05, e=128, d=256, c=512, attention_win_size=3,
                test_data='harvard_sentences.txt', vocab="PE abcdefghijklmnopqrstuvwxyz'.?", max_N=180,
                max_T=210, lr=0.001, logdir="logdir/LJ01", sampledir='samples', B=32, num_iterations=2000000)
    for k, v in want.items():
        assert getattr(hp, k) == v, k
    assert len(hp.vocab) == 32


def test_text_adaptor_harvard_sentence_1():
    # SURVEY.md 8(d) config 1: "the birch canoe slid on the smooth planks.E" = 43 ids padded to 180
    L = load_data("synthesize", os.path.join(ROOT, "harvard_sentences.txt"))
    assert L.shape == (20, hp.max_N) and L.dtype == np.int32
    c2i, i2c = load_vocab()
    s = "".join(i2c[i] for i in L[0][:43])
    assert s == "the birch canoe slid on the smooth planks.E"
    assert (L[0][43:] == 0).all() and L[0][42] == 1
    assert text_normalize("Héllo,  WORLD!") == "hello world "


def test_scope_names_are_tf_variable_names():
    shapes = arch.param_shapes()
    assert shapes["Text2Mel/TextEnc/embed_1/lookup_table"] == (32, 128)
    assert shapes["Text2Mel/TextEnc/C_2/conv1d/kernel"] == (1, 128, 512)
    assert shapes["Text2Mel/TextEnc/HC_15/conv1d/kernel"] == (1, 512, 1024)
    assert shapes["Text2Mel/AudioEnc/HC_13/H2/gamma"] == (256,)
    assert shapes["Text2Mel/AudioDec/C_11/normalize/beta"] == (80,)
    assert shapes["SSRN/D_4/conv2d_transpose/kernel"] == (1, 3, 512, 512)
    assert shapes["SSRN/C_16/conv1d/kernel"] == (1, 1025, 1025)
    assert "SSRN/C_17/conv1d/kernel" not in shapes          # networks.py:285-290: counter not advanced


def test_library_exports_every_declared_symbol():
    """The built .so must export exactly what include/dctts.h declares (no compute calls here)."""
    header = open(os.path.join(ROOT, "include", "dctts.h")).read()
    declared = set(re.findall(r"\b(dctts_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    lib.dctts_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.dctts_version()


def test_no_cpu_fallback():
    """Without a CUDA device the product refuses to run instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dc_tts_b200.engine import DcttsError, Engine
    with pytest.raises(DcttsError):
        Engine(0)
    lib = _lib.load()
    st = _lib.HParams(32, 128, 256, 512, 80, 2048, 180, 210, 3, 4)
    h = _lib.Handle()
    assert lib.dctts_create(ctypes.byref(st), 0, ctypes.byref(h)) != 0
    assert lib.dctts_last_error(None)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "dc_tts_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("the oracle", "").replace("oracle tests", ""), f
