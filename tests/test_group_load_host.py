"""Host-side checks of the group's file load (no GPU needed): the rank-info struct as ctypes sees it, and the entry points
refuse a null handle before touching a device."""
import ctypes as C


def test_rank_info_layout():
    from lantern_b200 import api
    assert C.sizeof(api.GroupRankInfo) == 56  # 2 ints + 6 uint64, x86-64 SysV
    assert api.GroupRankInfo.rows_begin.offset == 8 and api.GroupRankInfo.bytes_mailbox.offset == 48


def test_null_group_handle():
    from lantern_b200 import api
    L = api.lib()
    o = api.init_options(16)
    buf = (C.c_uint8 * 136)()
    for name, args in (("lb200_group_load_buffer", (None, C.byref(o), buf, 136, 0, 0, 0)),
                       ("lb200_group_load", (None, C.byref(o), b"/nonexistent", 0, 0, 0)),
                       ("lb200_group_rank_info", (None, 0, C.byref(api.GroupRankInfo())))):
        err = C.c_char_p()
        getattr(L, name)(*args, C.byref(err))
        assert err.value == b"null group handle", (name, err.value)
