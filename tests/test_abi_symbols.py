"""The C-ABI library loads on a machine WITHOUT a GPU and exports exactly the symbols include/newsrec_b200.h
declares; the ctypes table lists every one of them.  No compute calls here."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "newsrec_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nr_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_boundary():
    syms = declared_symbols()
    for must in ("nr_mhsa_encoder_fwd", "nr_mhsa_encoder_bwd", "nr_cnn_encoder_fwd", "nr_cnn_encoder_bwd", "nr_gru_fwd", "nr_gru_bwd",
                 "nr_additive_attention_fwd", "nr_dot_score_fwd", "nr_gather_rows", "nr_linear", "nr_gemm_tn", "nr_last_error"):
        assert must in syms, must


def test_library_exports_every_declared_symbol():
    import newsrec_b200
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built (python __graft_entry__.py build)")
    lib = ctypes.CDLL(newsrec_b200.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, missing


def test_ctypes_table_matches_header():
    import newsrec_b200
    assert sorted(newsrec_b200.SIGNATURES.keys()) == declared_symbols()


def test_version_and_error_string_without_gpu():
    import newsrec_b200
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built")
    lib = newsrec_b200.load_library()
    assert lib.nr_version() == 1
    assert isinstance(lib.nr_last_error(), bytes)
    # argument validation happens before any launch: a null-pointer call fails cleanly without a device
    assert lib.nr_dot_score_fwd(None, None, 1, 1, 1, None, None) == -1
    assert b"null operand" in lib.nr_last_error()


def test_struct_layouts_match_the_header_field_order():
    import newsrec_b200 as nb
    text = open(HEADER).read()
    for cname, cls in (("nr_mhsa_encoder_fwd_args", nb.MhsaEncoderFwdArgs), ("nr_mhsa_encoder_bwd_args", nb.MhsaEncoderBwdArgs),
                       ("nr_cnn_encoder_fwd_args", nb.CnnEncoderFwdArgs), ("nr_cnn_encoder_bwd_args", nb.CnnEncoderBwdArgs),
                       ("nr_gru_fwd_args", nb.GruFwdArgs), ("nr_gru_bwd_args", nb.GruBwdArgs),
                       ("nr_gemm_store_args", nb.GemmStoreArgs)):
        end = re.search(r"\}\s*" + cname + r"\s*;", text).start()
        start = text.rfind("typedef struct {", 0, end) + len("typedef struct {")
        body = re.sub(r"/\*.*?\*/", "", text[start:end], flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):
                names.append(re.findall(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", part.strip())[0])
        assert names == [f[0] for f in cls._fields_], (cname, names, [f[0] for f in cls._fields_])
