"""CPU checks of the device-resident frame store: the argument checks of osvos_affine_warp_u8_indexed (csrc/frames.cu),
the ``train_parent.py --cache`` refusals, and the shard plan by which R ranks split the decoding (davis.shard_plan)."""
import ctypes

import pytest

ADDR = 1 << 20                                           # placeholder device address, never dereferenced


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


def test_affine_warp_u8_indexed_checks_arguments_first(lib):
    mats = (ctypes.c_double * 12)(1, 0, 0, 0, 1, 0, 1, 0, 0, 0, 1, 0)
    flips = (ctypes.c_int * 2)(0, 1)
    ok = dict(image_src=ADDR, label_src=ADDR, label_stats=ADDR, image_dst=ADDR, label_dst=ADDR, mats=mats,
              index=(0, 3))

    def call(n=2, n_store=4, h=8, w=8, **kw):
        a = dict(ok, **kw)
        index = None if a["index"] is None else (ctypes.c_int * len(a["index"]))(*a["index"])
        return lib.osvos_affine_warp_u8_indexed(a["image_src"], a["label_src"], a["label_stats"], a["image_dst"],
                                                a["label_dst"], index, a["mats"], flips, n, n_store, h, w, 104.0,
                                                116.0, 122.0, None)
    for kw, rejected_by in [(dict(index=None), "index_host != nullptr"),
                            (dict(mats=None), "inv_matrices_host != nullptr"),
                            (dict(index=(0, -1)), "index_host[i] >= 0"),
                            (dict(index=(4, 0)), "index_host[i] < n_store"),
                            (dict(index=(0,), n=1, n_store=0), "n_store > 0"),
                            (dict(index=(0,), n=1, n_store=-3), "n_store > 0"),
                            (dict(n=0), "n > 0"), (dict(n=-1), "n > 0"),
                            (dict(image_src=None, label_src=None, label_stats=None), "image_store != nullptr"),
                            (dict(image_dst=None), "image_dst == nullptr"),
                            (dict(image_src=None), "image_dst == nullptr"),
                            (dict(label_stats=None), "label_stats == nullptr"),
                            (dict(label_dst=None), "label_dst == nullptr"),
                            (dict(label_src=None), "label_dst == nullptr"),
                            (dict(h=0), "h > 0"), (dict(w=32768), "w < 32768")]:
        assert call(**kw) == 1, kw
        msg = lib.osvos_last_error()
        assert b"invalid argument" in msg and rejected_by.encode() in msg, (kw, msg)


@pytest.mark.parametrize("extra,message", [(["--synthetic"], "--synthetic"), ([], "--loader reference"),
                                           (["--loader", "reference"], "--loader reference"),
                                           (["--synthetic", "--loader", "native"], "--synthetic")])
def test_parent_cache_needs_the_native_loader(extra, message, capsys):
    import train_parent
    with pytest.raises(SystemExit):
        train_parent.parse(["--cache", "device"] + extra)
    err = capsys.readouterr().err
    assert "--cache device" in err and message in err


def test_parent_cache_parses():
    import train_parent
    a = train_parent.parse(["--cache", "device", "--loader", "native"])
    assert a.cache == "device" and a.loader == "native"
    assert train_parent.parse([]).cache == "none"
    assert train_parent.parse(["--synthetic"]).cache == "none"
    with pytest.raises(SystemExit):
        train_parent.parse(["--cache", "host", "--loader", "native"])


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_shard_plan_decodes_each_frame_once(world):
    from osvos_pytorch_b200.davis import shard, shard_plan
    # sizes in runs and alternations, as DAVIS sequences of different sizes would give them
    sizes = [(33, 45)] * 7 + [(97, 131)] * 3 + [(33, 45), (97, 131)] * 4 + [(10, 12)] * 2
    n = len(sizes)
    decoded = sorted(i for r in range(world) for i in shard(n, world, r))
    assert decoded == list(range(n))
    plan = shard_plan(sizes, world)
    assert [size for size, _, _ in plan] == [(33, 45), (97, 131), (10, 12)]
    seen = []
    for size, pad, members in plan:
        assert len(members) == world
        assert pad == max(len(m) for m in members)
        slots = set()
        for r, m in enumerate(members):
            assert m == [i for i in shard(n, world, r) if sizes[i] == size]        # in the rank's decode order
            slots.update(r * pad + j for j in range(len(m)))
            seen += m
        assert len(slots) == sum(len(m) for m in members) and max(slots) < world * pad
    assert sorted(seen) == list(range(n))
    if world == 1:                                       # one rank: dataset order, no padding
        assert [members[0] for _, _, members in plan] == [[i for i in range(n) if sizes[i] == s] for s, _, _ in plan]
        assert all(pad == len(members[0]) for _, pad, members in plan)
