"""ctypes binding of libbinder_b200.so (include/binder_b200.h).  There is no CPU fallback:
a missing library or a missing CUDA device is an error, never a silent different path."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, 'libbinder_b200.so')

# name -> (restype, argtypes); every symbol include/binder_b200.h declares
_c = ctypes
SYMBOLS = {
    'bb_strerror': (_c.c_char_p, [_c.c_int]),
    'bb_last_cuda_error': (_c.c_char_p, []),
    'bb_abi_version': (_c.c_int, []),
    'bb_zone_build': (_c.c_void_p, [_c.c_char_p, _c.c_size_t, _c.c_char_p, _c.POINTER(_c.c_int)]),
    'bb_zone_build_shard': (_c.c_void_p, [_c.c_char_p, _c.c_size_t, _c.c_char_p, _c.c_uint32, _c.c_uint32,
                                          _c.POINTER(_c.c_int)]),
    'bb_zone_free': (None, [_c.c_void_p]),
    'bb_zone_apply': (_c.c_int, [_c.c_void_p, _c.c_char_p, _c.c_size_t]),
    'bb_zone_probe': (_c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_char_p, _c.c_uint32] + [_c.c_void_p] * 4 + [_c.c_uint32, _c.c_void_p]),
    'bb_engine_apply_update': (_c.c_int, [_c.c_void_p, _c.c_void_p]),
    'bb_zone_stat': (_c.c_uint64, [_c.c_void_p, _c.c_int]),
    'bb_engine_create': (_c.c_void_p, [_c.c_void_p, _c.POINTER(_c.c_int)]),
    'bb_engine_destroy': (None, [_c.c_void_p]),
    'bb_engine_swap_zone': (_c.c_int, [_c.c_void_p, _c.c_void_p]),
    'bb_engine_is_ready': (_c.c_int, [_c.c_void_p]),
    'bb_engine_set_recursion_filter': (_c.c_int, [_c.c_void_p, _c.c_char_p, _c.c_void_p, _c.c_uint32, _c.c_int]),
    'bb_resolve_batch': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint64, _c.c_uint32,
                                    _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                    _c.c_void_p]),
    'bb_engine_slots': (_c.c_int, [_c.c_void_p]),
    'bb_shard_use_exchange_buffers': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p]),
    'bb_shard_exchange_bytes': (_c.c_size_t, [_c.c_void_p]),
    'bb_shard_exchange_set': (_c.c_uint32, [_c.c_void_p]),
    'bb_shard_region_layout': (None, [_c.c_void_p, _c.c_void_p]),
    'bb_engine_set_kernel_profile': (_c.c_int, [_c.c_void_p, _c.c_int]),
    'bb_engine_max_batch': (_c.c_uint32, [_c.c_void_p]),
    'bb_engine_max_batch_bytes': (_c.c_uint32, [_c.c_void_p]),
    'bb_resolve_submit': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint64,
                                     _c.c_uint32, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                     _c.c_void_p, _c.c_void_p]),
    'bb_resolve_wait': (_c.c_int, [_c.c_void_p, _c.c_int]),
    'bb_resolve_batch_ex': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint64, _c.c_uint32,
                                       _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                       _c.c_void_p, _c.c_uint32]),
    'bb_resolve_submit_ex': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint64,
                                        _c.c_uint32, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                        _c.c_void_p, _c.c_void_p, _c.c_uint32]),
    'bb_resolve_batch_device': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint64,
                                           _c.c_uint32, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p,
                                           _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    'bb_resolve_batch_device_ex': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint64,
                                              _c.c_uint32, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p,
                                              _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32]),
    'bb_relay_batch': (_c.c_int, [_c.c_void_p] * 5 + [_c.c_uint32, _c.c_uint32, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p,
                                                      _c.c_void_p]),
    'bb_relay_batch_device': (_c.c_int, [_c.c_void_p] * 5 + [_c.c_uint32, _c.c_uint32, _c.c_void_p, _c.c_uint32] + [_c.c_void_p] * 5),
    'bb_log_batch': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint32] + [_c.c_void_p] * 3 + [_c.c_uint32, _c.c_void_p, _c.c_uint32] +
                     [_c.c_void_p] * 4),
    'bb_log_batch_device': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint32] + [_c.c_void_p] * 4 + [_c.c_uint32, _c.c_void_p,
                                                                                                      _c.c_uint32] + [_c.c_void_p] * 6),
    'bb_engine_set_recursion_upstreams': (_c.c_int, [_c.c_void_p] * 4 + [_c.c_uint32]),
    'bb_forward_batch': (_c.c_int, [_c.c_void_p] * 3 + [_c.c_uint32, _c.c_uint64, _c.c_void_p, _c.c_uint32] + [_c.c_void_p] * 4),
    'bb_forward_batch_device': (_c.c_int, [_c.c_void_p] * 5 + [_c.c_uint32, _c.c_uint64, _c.c_void_p, _c.c_uint32] +
                                [_c.c_void_p] * 5 + [_c.c_uint32] + [_c.c_void_p] * 3),
    'bb_match_upstreams': (_c.c_int, [_c.c_void_p] * 5 + [_c.c_uint32] + [_c.c_void_p] * 3 + [_c.c_uint32, _c.c_uint64,
                                                                                              _c.c_void_p, _c.c_uint32, _c.c_void_p]),
    'bb_match_upstreams_device': (_c.c_int, [_c.c_void_p] * 5 + [_c.c_uint32] + [_c.c_void_p] * 4 +
                                  [_c.c_uint32, _c.c_uint64, _c.c_void_p, _c.c_uint32] + [_c.c_void_p] * 3),
    'bb_engine_launch_count': (_c.c_uint64, [_c.c_void_p]),
    'bb_engine_launch_epoch': (_c.c_uint32, [_c.c_void_p]),
    'bb_engine_set_stage_log': (None, [_c.c_void_p, _c.c_void_p]),
    'bb_shard_create': (_c.c_void_p, [_c.c_void_p, _c.c_uint32, _c.c_uint32, _c.c_uint32, _c.c_uint32, _c.POINTER(_c.c_int)]),
    'bb_shard_destroy': (None, [_c.c_void_p]),
    'bb_shard_ipc_handle_size': (_c.c_uint32, []),
    'bb_shard_region_capacity': (_c.c_uint32, [_c.c_void_p]),
    'bb_shard_get_ipc_handle': (_c.c_int, [_c.c_void_p, _c.c_void_p]),
    'bb_shard_open_peers': (_c.c_int, [_c.c_void_p, _c.c_void_p]),
    'bb_shard_route_push': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint32, _c.c_void_p]),
    'bb_shard_route_push_ex': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_uint32, _c.c_uint32,
                                          _c.c_void_p]),
    'bb_shard_resolve': (_c.c_int, [_c.c_void_p, _c.c_uint64, _c.c_int, _c.c_void_p]),
    'bb_shard_fetch': (_c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                  _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    'bb_shard_host_results': (_c.c_int, [_c.c_void_p, _c.c_int]),
    'bb_shard_results': (_c.c_int, [_c.c_void_p, _c.c_uint32] + [_c.c_void_p] * 9),
    'bb_frames_parse': (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                   _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p]),
    'bb_frames_build': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint32,
                                   _c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bb_backend_create': (_c.c_void_p, [_c.c_void_p, _c.c_uint32, _c.POINTER(_c.c_int)]),
    'bb_backend_destroy': (None, [_c.c_void_p]),
    'bb_backend_feed': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_uint64, _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    'bb_backend_relay': (_c.c_int, [_c.c_void_p] * 7 + [_c.c_uint32, _c.c_void_p, _c.c_void_p]),
    'bb_backend_stat': (_c.c_uint64, [_c.c_void_p, _c.c_int]),
    'bb_query_log_backend_enable': (_c.c_int, [_c.c_void_p, _c.c_int]),
    'bb_query_log_backend': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p]),
    'bb_tcp_hub_create': (_c.c_void_p, [_c.c_void_p, _c.c_uint32, _c.POINTER(_c.c_int)]),
    'bb_tcp_hub_destroy': (None, [_c.c_void_p]),
    'bb_tcp_hub_open': (_c.c_int, [_c.c_void_p, _c.c_void_p]),
    'bb_tcp_hub_feed': (_c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_size_t]),
    'bb_tcp_hub_eof': (_c.c_int, [_c.c_void_p, _c.c_uint32]),
    'bb_tcp_hub_flush': (_c.c_int, [_c.c_void_p, _c.c_uint64, _c.c_void_p]),
    'bb_tcp_hub_output': (_c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    'bb_tcp_hub_consume': (_c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_size_t]),
    'bb_tcp_hub_close': (_c.c_int, [_c.c_void_p, _c.c_uint32]),
    'bb_tcp_hub_relay': (_c.c_int, [_c.c_void_p] * 6 + [_c.c_uint32]),
    'bb_tcp_hub_peer': (_c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_void_p, _c.c_void_p]),
    'bb_tcp_hub_stat': (_c.c_uint64, [_c.c_void_p, _c.c_int]),
    'bb_query_log_tcp_hub_enable': (_c.c_int, [_c.c_void_p, _c.c_int]),
    'bb_query_log_tcp_hub': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p]),
    'bb_host_alloc': (_c.c_void_p, [_c.c_size_t]),
    'bb_host_free': (None, [_c.c_void_p]),
}


class EngineOpts(ctypes.Structure):
    _fields_ = [('dns_domain', _c.c_char_p), ('datacenter_name', _c.c_char_p), ('recursion', _c.c_int32),
                ('device', _c.c_int32), ('max_batch', _c.c_uint32), ('max_batch_bytes', _c.c_uint32),
                ('ordered_output', _c.c_int32)]


_lib = None


def lib():
    """Load (once) and type the shared library.  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise RuntimeError('binder_b200: %s is missing — run `python -m binder_b200.build` '
                               '(there is no CPU fallback)' % SO_PATH)
        L = ctypes.CDLL(SO_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class BinderError(RuntimeError):
    def __init__(self, code):
        L = lib()
        msg = L.bb_strerror(code).decode()
        if code == -3:
            msg += ': ' + L.bb_last_cuda_error().decode()
        RuntimeError.__init__(self, 'binder_b200 error %d: %s' % (code, msg))
        self.code = code


def check(code):
    if code != 0:
        raise BinderError(code)
