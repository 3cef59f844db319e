"""ctypes binding of libp2p_b200.so (C ABI in include/p2p_b200.h).

There is no fallback: if the CUDA library is missing or fails to load, importing
anything that needs it raises.  Build it with ``python -m patch2pix_b200.build``
(or ``__graft_entry__.build()``).
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libp2p_b200.so')
_lib = None


class BN(C.Structure):
    _fields_ = [('weight', C.c_void_p), ('bias', C.c_void_p), ('running_mean', C.c_void_p), ('running_var', C.c_void_p)]


class RegressorWeights(C.Structure):
    _fields_ = [('conv0_weight', C.c_void_p), ('conv1_bn', BN), ('conv2_weight', C.c_void_p), ('conv3_bn', BN),
                ('fc0_weight', C.c_void_p), ('fc0_bias', C.c_void_p), ('fc1_bn', BN),
                ('fc3_weight', C.c_void_p), ('fc3_bias', C.c_void_p), ('fc4_bn', BN),
                ('fc6_weight', C.c_void_p), ('fc6_bias', C.c_void_p), ('bn_eps', C.c_float)]


_P, _I, _LL, _F = C.c_void_p, C.c_int, C.c_longlong, C.c_float
_SIGNATURES = {
    'p2p_last_error': (C.c_char_p, []),
    'p2p_version': (_I, []),
    'p2p_create': (_I, [_I, C.POINTER(_P)]),
    'p2p_destroy': (_I, [_P]),
    'p2p_set_ncn_weights': (_I, [_P, _P, _P, _P, _P]),
    'p2p_set_regressor_weights': (_I, [_P, _I, C.POINTER(RegressorWeights)]),
    'p2p_set_option': (_I, [_P, C.c_char_p, _I]),
    'p2p_get_option': (_I, [_P, C.c_char_p, C.POINTER(_I)]),
    'p2p_launch_count': (_I, [_P, C.POINTER(_LL)]),
    'p2p_coarse': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'p2p_coarse_nhwc16': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'p2p_delta_unpack': (_I, [_P, _P, _LL, _I, _P, _P, _P, _P, _P]),
    'p2p_delta_pack': (_I, [_P, _P, _P, _P, _P, _LL, _I, _P, _P]),
    'p2p_mutual_matching': (_I, [_P, _P, _I, _I, _P, _P]),
    'p2p_neigh_consensus': (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    'p2p_set_nc_stack_weights': (_I, [_P, _I, _P, _P, _P, _P, _I]),
    'p2p_nc_stack': (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    'p2p_ncnet_coarse': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'p2p_proposals': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'p2p_proposals_topk': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    'p2p_unique_rows': (_I, [_P, _P, _I, _I, _P, _F, _P, _P, _P]),
    'p2p_select_anchor': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P]),
    'p2p_refine_prepare': (_I, [_P, C.POINTER(_P), C.POINTER(_P), _I, _I, _I, _I, _P]),
    'p2p_refine_prepare_nhwc16': (_I, [_P, C.POINTER(_P), C.POINTER(_P), _I, _I, _I, _I, _P]),
    'p2p_refine': (_I, [_P, _I, _P, _I, _I, _P, _P, _P]),
    'p2p_refine_taps': (_I, [_P, C.POINTER(C.c_int32), C.POINTER(_F), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'p2p_finalize_matches': (_I, [_P, _P, _P, _P, _I, _F, C.POINTER(C.c_double), _P, _P]),
    'p2p_preprocess_image': (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P]),
    'p2p_preprocess_image_gray': (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P]),
    'p2p_profile_read': (_I, [_P, C.POINTER(C.c_float), C.POINTER(_I), _I]),
    'p2p_test_gemm': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    'p2p_tile_trace_read': (_I, [_P, _I, C.POINTER(_I), C.POINTER(_I), _P, _I]),
    'p2p_find_model': (_I, [_P, _I, _P, _I, _I, _P, C.c_double, C.c_double, _I, C.c_ulonglong, _P, _P, _P, _P]),
    'p2p_sampson_distance': (_I, [_P, _P, _I, _I, _P, _P, _P]),
    'p2p_epipolar_histograms': (_I, [_P, _P, _I, _I, _P, _I, C.POINTER(C.c_double), _P, C.POINTER(C.c_double), _I, _P,
                                     _P]),
    'p2p_homography_errors': (_I, [_P, _P, _I, _I, _P, C.POINTER(C.c_double), _P, _I, _I, C.POINTER(C.c_double), _I,
                                   _P, _P, _P]),
    'p2p_overlap_scores': (_I, [_P, _P, _P, C.POINTER(C.c_int64), _I, _I, _P, _P, _P, _P]),
    'p2p_test_hypotheses': (_I, [_P, _I, _P, _I, _I, C.c_double, C.c_ulonglong, _I, _P, _P, _P]),
    'p2p_test_degeneracy': (_I, [_P, _P, _I, _I, C.c_double, C.c_ulonglong, _I, _P, _P, _P]),
    'p2p_find_essential': (_I, [_P, _P, _I, _I, _P, _P, C.c_double, C.c_double, _I, C.c_ulonglong, _P, _P, _P, _P]),
    'p2p_recover_pose': (_I, [_P, _P, _I, _I, _P, _P, _P, _P, C.c_double, _P, _P, _P, _P]),
    'p2p_test_essential_hypotheses': (_I, [_P, _P, _I, _I, _P, C.c_double, C.c_ulonglong, _I, _P, _P, _P]),
    'p2p_find_model_batch': (_I, [_P, _I, _P, _I, _P, C.POINTER(C.c_int64), _I, _P, C.c_double, C.c_double, _I,
                                  C.c_ulonglong, _P, _P, _P, _P]),
    'p2p_find_essential_batch': (_I, [_P, _P, _I, _P, C.POINTER(C.c_int64), _I, _P, _P, C.c_double, C.c_double, _I,
                                      C.c_ulonglong, _P, _P, _P, _P]),
    'p2p_find_essential_batch_th': (_I, [_P, _P, _I, _P, C.POINTER(C.c_int64), _I, _P, _P, _P, C.c_double, _I,
                                         C.c_ulonglong, _P, _P, _P, _P]),
    'p2p_relpose_errors_batch': (_I, [_P, _P, _I, _P, C.POINTER(C.c_int64), _I, _P, _P, _P, _P, _P,
                                      C.POINTER(C.c_double), _I, _P, _I, _P]),
    'p2p_recover_pose_batch': (_I, [_P, _P, _I, _P, C.POINTER(C.c_int64), _I, _P, _P, _P, _P, C.c_double, _P, _P, _P,
                                    _P]),
    'p2p_batch_chunk_pairs': (_I, [_P, _I, C.POINTER(_I)]),
    'p2p_find_absolute_pose_batch': (_I, [_P, _P, _I, _P, C.POINTER(C.c_int64), _I, _P, _P, C.c_double, _P, C.c_double,
                                          _I, C.c_ulonglong, _P, _P, _P, _P]),
    'p2p_lift_scan': (_I, [_P, _P, _I, _I, C.POINTER(C.c_double), _P, _I, _I, _P, _P, _I, _LL, _P, _P]),
    'p2p_test_absolute_pose_hypotheses': (_I, [_P, _P, _I, _I, C.POINTER(C.c_double), C.c_double, C.c_ulonglong, _I, _P,
                                               _P, _P]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)
PROF_KINDS = ('l2norm', 'corr', 'mutual', 'nc', 'proposals', 'prep', 'gather_mid', 'conv1_mid', 'conv2_mid', 'fc_mid',
              'gather_fine', 'conv1_fine', 'conv2_fine', 'fc_fine', 'gather_band', 'conv1_band', 'conv2_band', 'fc_band',
              'flag')


def load():
    """Load (once) and return the ctypes library.  Raises if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f'{LIB_PATH} not found: the CUDA extension is required (no CPU fallback). '
                               f'Build it with `python -m patch2pix_b200.build`.')
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)      # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        msg = load().p2p_last_error()
        raise RuntimeError(f'libp2p_b200 error {rc}: {msg.decode() if msg else "?"}')


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Handle:
    """Owns one p2p_handle_t on `device` (packed weights + scratch)."""

    def __init__(self, device):
        device = torch.device(device)
        if device.type != 'cuda':
            raise RuntimeError('patch2pix_b200 runs on CUDA (sm_90a) devices only; got device ' + str(device))
        self.device = torch.device('cuda', device.index if device.index is not None else torch.cuda.current_device())
        self.lib = load()
        h = C.c_void_p()
        check(self.lib.p2p_create(self.device.index, C.byref(h)))
        self.h = h
        # P2P_OPTIONS="nc_impl=0,mid_band=0": option overrides for A/B measurements (bench.py)
        for kv in filter(None, os.environ.get('P2P_OPTIONS', '').split(',')):
            k, _, v = kv.partition('=')
            self.set_option(k.strip(), int(v))

    def __del__(self):
        try:
            if getattr(self, 'h', None):
                self.lib.p2p_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_option(self, key, value):
        check(self.lib.p2p_set_option(self.h, key.encode(), int(value)))

    def get_option(self, key):
        v = C.c_int()
        check(self.lib.p2p_get_option(self.h, key.encode(), C.byref(v)))
        return v.value

    def tile_traces(self):
        """[(tag, stamps)] of the launches traced since option 'tile_trace' was set: stamps is [tiles][8] uint64
        (p2p_tile_trace_read), rows of tiles the launch did not have are dropped.  Synchronises."""
        import numpy as np
        out = []
        for i in range(self.get_option('tile_traces')):
            tag, tiles = C.c_int(), C.c_int()
            check(self.lib.p2p_tile_trace_read(self.h, i, C.byref(tag), C.byref(tiles), None, 0))
            buf = np.zeros((tiles.value, 8), dtype=np.uint64)
            check(self.lib.p2p_tile_trace_read(self.h, i, C.byref(tag), C.byref(tiles), buf.ctypes.data, tiles.value))
            out.append((tag.value, buf[buf[:, 6] != 0]))
        return out

    def launch_count(self):
        v = C.c_longlong()
        check(self.lib.p2p_launch_count(self.h, C.byref(v)))
        return v.value

    def stream(self):
        return stream_ptr(self.device)

    def profile_read(self):
        """-> {kind name: (total ms, launch groups)} since the last read (needs option profile=1)."""
        n = len(PROF_KINDS)
        ms = (C.c_float * n)()
        cnt = (C.c_int * n)()
        check(self.lib.p2p_profile_read(self.h, ms, cnt, n))
        return {PROF_KINDS[i]: (ms[i], cnt[i]) for i in range(n)}


_default_handles = {}


def default_handle(device):
    """Weight-less per-device handle for the stateless ops (filter_coarse, proposals, ...)."""
    device = torch.device(device)
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _default_handles:
        _default_handles[idx] = Handle(torch.device('cuda', idx))
    return _default_handles[idx]
