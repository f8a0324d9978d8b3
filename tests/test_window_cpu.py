"""CPU tier for the sliding-window kernels (csrc/window.cu): every entry point rejects bad arguments with
SEMSEG_E_INVALID and a message naming it before any CUDA call, so no GPU is needed."""
import ctypes

from semseg_b200 import _lib

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _ints(*v):
    return (ctypes.c_int * len(v))(*v)


def _err():
    return _lib.load().semseg_last_error()


def test_window_scores_validates_arguments():
    lib = _lib.load()
    # semseg_window_scores(logits, pitch, G, h, w, C, flip, out, crop_h, crop_w, stream); 9x9 logits -> 65x65 crop
    assert lib.semseg_window_scores(None, 7, 1, 9, 9, 7, 1, P, 65, 65, None) == -1
    assert b"window_scores" in _err() and b"null" in _err()
    assert lib.semseg_window_scores(P, 7, 1, 9, 9, 7, 1, None, 65, 65, None) == -1
    assert lib.semseg_window_scores(P, 257, 1, 9, 9, 257, 1, P, 65, 65, None) == -1      # more than 256 classes
    assert b"window_scores" in _err() and b"C<=256" in _err()
    assert lib.semseg_window_scores(P, 6, 1, 9, 9, 7, 1, P, 65, 65, None) == -1          # pitch < C
    assert b"window_scores" in _err()
    assert lib.semseg_window_scores(P, 7, 1, 9, 9, 7, 2, P, 65, 65, None) == -1          # flip must be 0 or 1
    assert lib.semseg_window_scores(P, 7, 0, 9, 9, 7, 1, P, 65, 65, None) == -1          # no crops
    assert lib.semseg_window_scores(P, 7, 1, 9, 9, 7, 1, P, 64, 65, None) == -1          # crop != 8(h-1)+1
    assert b"window_scores" in _err() and b"8(h-1)+1" in _err()
    assert lib.semseg_window_scores(P, 7, 1, 9, 9, 7, 0, P, 65, 73, None) == -1


def test_window_accumulate_validates_arguments():
    lib = _lib.load()
    ys, xs = _ints(0, 44, 45), _ints(0, 44)        # crop 65 on a padded 110 x 109 image

    def call(scores=P, C=7, ys=ys, ny=3, xs=xs, nx=2, full=(110, 109), top=0, left=0, img=(110, 109), canvas=P):
        return lib.semseg_window_accumulate(scores, C, 65, 65, ys, ny, xs, nx, full[0], full[1], top, left, img[0],
                                            img[1], canvas, None)

    assert call(scores=None) == -1 and b"window_accumulate" in _err() and b"null" in _err()
    assert call(canvas=None) == -1
    assert call(ys=None) == -1 and b"window_accumulate" in _err()
    assert call(C=0) == -1 and b"window_accumulate" in _err()
    assert call(img=(111, 109)) == -1                                  # image larger than the padded extent
    assert call(top=1) == -1                                           # un-padded window leaves the padded image
    assert call(ys=_ints(1, 44, 45)) == -1 and b"out of range" in _err()
    assert call(ys=_ints(0, 44, 46)) == -1 and b"out of range" in _err()     # last crop past the border
    assert call(ys=_ints(0, 45, 45)) == -1 and b"ascend" in _err()
    assert call(ys=_ints(0, 40, 30, 45), ny=4) == -1 and b"ascend" in _err()
    assert call(ys=_ints(0, 45), ny=2, full=(130, 109), img=(130, 109)) == -1 and b"out of range" in _err()  # ends at 110
    assert call(ys=_ints(0, 66), ny=2, full=(131, 109), img=(131, 109)) == -1 and b"gaps" in _err()   # row 65 uncovered
    assert call(ny=0) == -1 and b"window_accumulate" in _err()
    assert call(ny=257) == -1 and b"window_accumulate" in _err()


def test_window_resize_add_validates_arguments():
    lib = _lib.load()
    # semseg_window_resize_add(canvas, C, Hi, Wi, total, Ho, Wo, stream)
    assert lib.semseg_window_resize_add(None, 7, 10, 10, P, 20, 20, None) == -1
    assert b"window_resize_add" in _err() and b"null" in _err()
    assert lib.semseg_window_resize_add(P, 7, 10, 10, None, 20, 20, None) == -1
    assert lib.semseg_window_resize_add(P, 0, 10, 10, P, 20, 20, None) == -1
    assert b"window_resize_add" in _err()
    assert lib.semseg_window_resize_add(P, 7, 0, 10, P, 20, 20, None) == -1
    assert lib.semseg_window_resize_add(P, 7, 10, 10, P, 20, 0, None) == -1
