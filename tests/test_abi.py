"""CPU tier: the C-ABI library loads and exports exactly the symbols include/semseg_b200.h declares, and the
ctypes binding lists every one of them (no compute calls: there is no GPU here)."""
import ctypes
import os
import re
import subprocess

import pytest

from semseg_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "semseg_b200.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(semseg_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_symbols():
    syms = header_symbols()
    assert "semseg_conv_fprop" in syms and "semseg_psamask_fwd" in syms and len(syms) >= 20


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in header_symbols():
        assert hasattr(lib, s), "library does not export %s" % s


def test_no_undeclared_exports():
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r" T (semseg_[a-z0-9_]+)", out)))
    assert exported == header_symbols()


def test_ctypes_binding_covers_header():
    assert sorted(_lib.SIGNATURES) == header_symbols()
    lib = _lib.load()
    assert lib.semseg_abi_version() == 3
    assert lib.semseg_launch_count() == 0 or lib.semseg_launch_count() > 0


def test_struct_layout_matches_header():
    """sizeof / offsets of the ABI structs as the C compiler sees them == the ctypes mirrors."""
    import tempfile
    prog = r'''
#include <stdio.h>
#include "semseg_b200.h"
#include <stddef.h>
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(semseg_conv_desc), sizeof(semseg_wgrad_desc), sizeof(semseg_pack_item),
         offsetof(semseg_pack_item, wp), offsetof(semseg_pack_item, Cout), offsetof(semseg_pack_item, tile0),
         offsetof(semseg_pack_item, tiles_ci));
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        a, b, c, o_wp, o_cout, o_tile0, o_tiles = map(int, subprocess.check_output([exe]).split())
    assert a == ctypes.sizeof(_lib.ConvDesc)
    assert b == ctypes.sizeof(_lib.WgradDesc)
    # the item table of semseg_pack_weights_multi is built by ctypes and read by the device code
    assert c == ctypes.sizeof(_lib.PackItem)
    assert (o_wp, o_cout, o_tile0, o_tiles) == (_lib.PackItem.wp.offset, _lib.PackItem.Cout.offset,
                                                _lib.PackItem.tile0.offset, _lib.PackItem.tiles_ci.offset)


def test_invalid_arguments_return_error_codes_without_gpu():
    lib = _lib.load()
    # argument validation happens before any CUDA call
    assert lib.semseg_psamask_fwd(3, None, None, 1, 1, 1, 1, 1, None) == -1
    assert b"psa_type" in lib.semseg_last_error()
    assert lib.semseg_psamask_fwd(0, ctypes.c_void_p(16), ctypes.c_void_p(16), 1, 2, 2, 4, 3, None) == -1
    assert b"odd" in lib.semseg_last_error()
    d = _lib.ConvDesc()
    assert lib.semseg_conv_fprop(ctypes.byref(d), None) == -1
    assert lib.semseg_conv_stats_rows(1, 8, 16, 64) == 4
    assert lib.semseg_iou_hist(ctypes.c_void_p(16), ctypes.c_void_p(16), 10, 0, 255, 1, ctypes.c_void_p(16), None) == -1
    assert b"iou_hist" in lib.semseg_last_error()
    assert lib.semseg_im2col3x3s2(ctypes.c_void_p(16), 8, 1, 9, 9, 4, ctypes.c_void_p(16), None) == -1
    assert b"im2col3x3s2" in lib.semseg_last_error()
    assert lib.semseg_pack_weights_multi(None, 1, 1, 9, None) == -1
    assert not hasattr(lib, "semseg_pack_weights")          # the one-launch packing is the only packing entry point


def test_round2_struct_layouts_match_header():
    """semseg_sgd_item / semseg_sgd_hyper (tables built by ctypes, read by device / host code of csrc/sgd.cu) and the
    grown conv / wgrad descriptors as the C compiler lays them out."""
    import tempfile
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "semseg_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(semseg_sgd_item), offsetof(semseg_sgd_item, n),
         offsetof(semseg_sgd_item, chunk0), sizeof(semseg_sgd_hyper), offsetof(semseg_sgd_hyper, weight_decay),
         offsetof(semseg_sgd_hyper, nesterov), offsetof(semseg_conv_desc, x_lo), offsetof(semseg_wgrad_desc, dy_lo));
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        v = list(map(int, subprocess.check_output([exe]).split()))
    assert v == [ctypes.sizeof(_lib.SgdItem), _lib.SgdItem.n.offset, _lib.SgdItem.chunk0.offset,
                 ctypes.sizeof(_lib.SgdHyper), _lib.SgdHyper.weight_decay.offset, _lib.SgdHyper.nesterov.offset,
                 _lib.ConvDesc.x_lo.offset, _lib.WgradDesc.dy_lo.offset]


def test_round2_entry_points_validate_before_any_cuda_call():
    """Fused PSA attention, bilinear resize, fused SGD, K-slice finish, split-aware elementwise ops: bad arguments come back
    as SEMSEG_E_INVALID with a message naming the entry point — no GPU needed, nothing is launched."""
    lib = _lib.load()
    P = ctypes.c_void_p(16)
    err = lambda: lib.semseg_last_error()      # noqa: E731
    # semseg_psa_attend(mode, psa_type, attn, a_pitch, feat, feat_lo, feat_pitch, stats, out, out_lo, out_pitch,
    #                   N, H, W, mH, mW, C, scale, stream)
    assert lib.semseg_psa_attend(2, 0, P, 9, P, None, 512, P, P, None, 512, 1, 3, 3, 3, 3, 512, 1.0, None) == -1
    assert b"mode" in err()
    assert lib.semseg_psa_attend(0, 0, P, 9, P, None, 256, P, P, None, 256, 1, 3, 3, 3, 3, 256, 1.0, None) == -1
    assert b"feature width must be 512" in err()
    assert lib.semseg_psa_attend(0, 0, P, 16, P, None, 512, P, P, None, 512, 1, 3, 3, 4, 4, 512, 1.0, None) == -1
    assert b"mask geometry" in err()                                  # even mask sizes (lib/psa/functions/psamask.py:14)
    assert lib.semseg_psa_attend(0, 0, P, 9, P, None, 512, P, P, None, 512, 1, 3, 200, 3, 3, 512, 1.0, None) == -1
    assert b"wider than 128" in err()
    assert lib.semseg_psa_attend(0, 0, P, 9, P, P, 512, P, P, None, 512, 1, 3, 3, 3, 3, 512, 1.0, None) == -1
    assert b"same storage form" in err()                              # split features with a plain output
    assert lib.semseg_psa_attend_bwd_attn(5, P, 9, P, P, None, 512, P, None, 512, P, None, 512, P, 1, 3, 3, 3, 3, 512, 1.0,
                                          None) == -1
    assert b"psa_type" in err()
    assert lib.semseg_psa_attend_bwd_attn(0, None, 9, P, P, None, 512, P, None, 512, P, None, 512, P, 1, 3, 3, 3, 3, 512,
                                          1.0, None) == -1
    assert b"psa_attend_bwd_attn" in err()
    assert lib.semseg_resize_bilinear_fwd(None, None, 64, 1, 4, 4, 64, 8, 8, P, None, 64, None) == -1
    assert b"resize_bilinear_fwd" in err()
    assert lib.semseg_resize_bilinear_fwd(P, None, 56, 1, 4, 4, 64, 8, 8, P, None, 64, None) == -1       # pitch < C
    assert b"pitch 56 is smaller than C = 64" in err()
    assert lib.semseg_resize_bilinear_bwd(P, P, 64, 1, 4, 4, 64, 8, 8, P, None, 64, None) == -1
    assert b"same storage form" in err()
    h = _lib.SgdHyper()
    assert lib.semseg_sgd_multi(None, None, 1, 1, ctypes.byref(h), None) == -1 and b"sgd_multi" in err()
    assert lib.semseg_sgd_multi(P, P, 0, 0, ctypes.byref(h), None) == -1
    assert lib.semseg_sgd_chunk_elems() > 0
    assert lib.semseg_conv_splitk_finish(None, 1, 0, 1, 1, 1, 64, 0, None, None, None, None, 64, None, None, 64, None,
                                         None) == -1
    assert b"conv_splitk_finish" in err()
    assert lib.semseg_add_act(None, None, 8, None, None, 8, None, None, 8, 1, 8, None) == -1 and b"add_act" in err()
    # bf16x3 accumulation-chain planning is pure host arithmetic: K blocks = taps * Cin / 64, at most 8 per slice
    assert lib.semseg_conv_k_slices(4096, 9, 8) == 72 and lib.semseg_conv_k_slices(64, 1, 8) == 1
    assert lib.semseg_conv_k_slices(256, 9, 8) == 5 and lib.semseg_conv_splitk_rows(4) >= 1


def test_peer_exchange_arguments_validated_before_any_cuda_call():
    """The SyncBN peer-exchange arguments (peer_bufs, world, rank, slot, slot_floats, seq_ptr) of both statistics entry
    points go through one check: a bad world, rank, slot size or peer pointer is SEMSEG_E_INVALID with a message, before
    anything is launched (no GPU here)."""
    lib = _lib.load()
    P = ctypes.c_void_p(16)
    c = 64
    peers = (ctypes.c_void_p * 8)(*([16] * 8))
    holey = (ctypes.c_void_p * 2)(16, None)
    nf = lib.semseg_bn_workspace_floats(64, c)
    assert nf > 0

    def finalize(bufs, world, rank, slot_floats, seq_ptr=P):
        # semseg_bn_finalize_partials(stats_partial, rows, C, gamma, beta, eps, momentum, running_mean, running_var,
        #                             mean_invstd, scale_shift, peer_bufs, world, rank, slot, slot_floats, seq_ptr, stream)
        return lib.semseg_bn_finalize_partials(P, 4, c, None, None, 1e-5, 0.1, None, None, P, P, bufs, world, rank, 0,
                                               slot_floats, seq_ptr, None)

    def bwd_reduce(bufs, world, rank, slot_floats, seq_ptr=P):
        # semseg_bn_bwd_reduce(dy, dy_lo, dy_pitch, y, y_lo, y_pitch, x, x_lo, x_pitch, mean_invstd, scale_shift, M, C,
        #                      relu, workspace, workspace_floats, sums, sums_total, peer_bufs, world, rank, slot,
        #                      slot_floats, seq_ptr, stream)
        return lib.semseg_bn_bwd_reduce(P, None, c, None, None, 0, P, None, c, P, None, 64, c, 0, P, nf, P, P, bufs,
                                        world, rank, 0, slot_floats, seq_ptr, None)

    for call, need in ((finalize, 3 * c), (bwd_reduce, 2 * c)):
        assert call(peers, 9, 0, need) == -1 and b"world 9" in lib.semseg_last_error()
        assert call(peers, 2, 2, need) == -1 and b"rank 2" in lib.semseg_last_error()
        assert call(peers, 2, 0, need - 1) == -1 and b"slot too small" in lib.semseg_last_error()
        assert call(holey, 2, 0, need) == -1 and b"null peer pointer 1" in lib.semseg_last_error()
        assert call(peers, 2, 0, need, None) == -1 and b"sequence" in lib.semseg_last_error()
