"""The run-parallel Cheetah decoder (cl_decode.cu) against its CPU model (tests/cl_model.cpp) round for round, on an H100 (pytest -m gpu).

Every input is decoded from the oracle's stream through decode_device_path 1 (parallel decoder only) and 0 (the in-order kernel queued
behind it), into exactly n bytes followed by a canary. The device's {rounds, settled, run walks after round 0} must equal the model's at
the run count the decoder picks for this device (tests/cl_decode_seams.py mirrors cd_pick_runs with the device's SM count), path 1 must be
exact wherever the model settles within the 40-round budget and report size 0 where it does not, and path 0 is always exact. Inputs: the
corpora planted at the decoder's own run seams, text, mixed and low-entropy data, and stretches of one repeated quad (zeros, spaces),
which need one round per run they cover."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
import planted
import cl_decode_seams as cds
from conftest import payload

pytestmark = pytest.mark.gpu
CANARY = 0xA5
MIB = 1 << 20
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    import density_b200
    return density_b200.load()


@pytest.fixture(scope="module")
def sms(torch_cuda):
    return torch_cuda.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return cds.build_model(tmp_path_factory.mktemp("cl_model"))


def _text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


INPUTS = {
    "planted12": lambda sms: cds.cl_decode_corpus(12 * MIB + 77, 3, num_sms=sms)[0],
    "planted33": lambda sms: cds.cl_decode_corpus(33 * MIB + 66, 4, num_sms=sms)[0],
    "dickens200k": lambda sms: planted.base_text(200003),
    "text33": lambda sms: _text(33 * MIB + 5),
    "mixed": lambda sms: payload("mixed", 5 * MIB + 3, seed=9),
    "low": lambda sms: payload("low", 5 * MIB + 1, seed=9),
    "zeros39": lambda sms: cds.zeros(39),
    "zeros40": lambda sms: cds.zeros(40),
    "zeros41": lambda sms: cds.zeros(41),
    "spaces": lambda sms: cds.spaces(),
    "zero_hole": lambda sms: cds.zero_hole(),
}
GIVE_UP = ("zeros41", "spaces", "zero_hole")
REPEATED = ("zeros39", "zeros40") + GIVE_UP
_cache = {}


def case(name, sms):
    """(data, oracle stream)"""
    if name not in _cache:
        data = INPUTS[name](sms)
        _cache[name] = (data, oracle.encode("cheetah", data))
    return _cache[name]


_model_cache = {}


def model_stats(model, name, sms, data, enc, per_sm=8):
    key = (name, sms, per_sm)
    if key not in _model_cache:
        out, st = cds.model_decode(model, enc, data.size, cds.pick_runs(enc.size, sms, per_sm))
        st["exact"] = bool(st["settled"]) and out.size == data.size and bool((out == data).all())
        _model_cache[key] = st
    return _model_cache[key]


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev_decode(torch, lib, enc, n, path, canary=64):
    """-> (rc, size, output, canary bytes after cap = n, milliseconds of the call on the device)"""
    import density_b200
    d_in = torch.from_numpy(enc).cuda()
    d_out = torch.full((n + canary,), CANARY, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    rc = lib.density_b200_decode_device_path(density_b200.codec.ALG_IDS["cheetah"], d_in.data_ptr(), enc.size, d_out.data_ptr(), n,
                                             d_sz.data_ptr(), _stream(torch), path)
    e1.record()
    torch.cuda.synchronize()
    m = int(d_sz.item())
    out = d_out.cpu().numpy()
    return rc, m, out[:max(m, 0)], out[n:], e0.elapsed_time(e1)


def rounds(lib):
    r4 = (ctypes.c_uint32 * 4)()
    assert lib.density_b200_cheetah_decode_rounds(r4) == 0
    return list(r4)


def first_diff(a, b):
    k = min(a.size, b.size)
    d = np.flatnonzero(a[:k] != b[:k])
    return int(d[0]) if d.size else k


@pytest.mark.parametrize("name", list(INPUTS))
def test_rounds_match_the_model(torch_cuda, lib, sms, model, name, record_property):
    torch = torch_cuda
    data, enc = case(name, sms)
    nruns = cds.pick_runs(enc.size, sms)
    st = model_stats(model, name, sms, data, enc)
    rc, m, got, tail, _ = dev_decode(torch, lib, enc, data.size, 1)
    gpu = rounds(lib)
    line = (f"{name}: {sms} SMs, {nruns} runs, stream {enc.size} B; GPU rounds {gpu[0]} settled {gpu[1]} walks after round 0 {gpu[2]}; "
            f"model rounds {st['rounds']} settled {st['settled']} walks {st['walks']} queued {st['queued']}")
    rc0, m0, got0, tail0, ms0 = dev_decode(torch, lib, enc, data.size, 0)
    line += f"; path 0 {ms0:.1f} ms"
    print(line)
    record_property("rounds", line)
    assert rc == 0 and rc0 == 0
    assert (tail == CANARY).all() and (tail0 == CANARY).all(), "wrote past the output capacity"
    assert m0 == data.size and (got0 == data).all(), f"path 0: first differing byte {first_diff(got0, data)}"
    assert gpu[3] == cds.MAX_ROUNDS
    assert (gpu[0], gpu[1], gpu[2]) == (st["rounds"], st["settled"], st["queued"]), line
    if st["settled"]:
        assert st["exact"] and m == data.size and (got == data).all(), f"path 1: size {m}, first differing byte {first_diff(got, data)}"
    else:
        assert m == 0, "path 1 reported a size for a stream whose rounds did not settle"
    if name.startswith("zeros"):
        assert gpu[0] == min(nruns, cds.MAX_ROUNDS) and nruns == int(name[5:])
    if name in REPEATED:
        assert (name in GIVE_UP) == (not st["settled"]), line


def test_sharded_decoder_world1_shares_the_budget(torch_cuda, lib, sms):
    """density_b200_decode_sharded_cheetah with one rank: the zero hole does not settle within the same 40 rounds and is refused; the
    planted corpus is accepted and exact."""
    torch = torch_cuda
    from density_b200 import sharded
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    try:
        for name, ok in (("zero_hole", False), ("planted12", True)):
            data, enc = case(name, sms)
            d_in = torch.from_numpy(enc).cuda()
            d_out = torch.full((data.size + 64,), CANARY, dtype=torch.uint8, device="cuda")
            d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
            d_fl = torch.zeros(1, dtype=torch.int32, device="cuda")
            rc = lib.density_b200_decode_sharded_cheetah(dec._h, d_in.data_ptr(), enc.size, d_out.data_ptr(), data.size, d_sz.data_ptr(),
                                                         d_fl.data_ptr(), None, _stream(torch))
            torch.cuda.synchronize()
            assert rc == 0
            assert (d_out[data.size:].cpu().numpy() == CANARY).all()
            if ok:
                assert int(d_fl.item()) == 0 and int(d_sz.item()) == data.size
                assert (d_out[:data.size].cpu().numpy() == data).all()
            else:
                assert int(d_fl.item()) != 0, name
    finally:
        dec.close()


_CHILD = r"""
import ctypes, json, sys
import numpy as np
import torch
import density_b200
lib = density_b200.load()
d = sys.argv[1]
res = {}
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
for name in (["planted33k", "text33"] if int(sys.argv[2]) else []):
    data, enc = np.load(f"{d}/{name}.npy"), np.load(f"{d}/{name}.enc.npy")
    d_in = torch.from_numpy(enc).cuda()
    d_out = torch.full((data.size + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_decode_device_path(density_b200.codec.ALG_IDS["cheetah"], d_in.data_ptr(), enc.size, d_out.data_ptr(), data.size,
                                             d_sz.data_ptr(), st, 1)
    torch.cuda.synchronize()
    r4 = (ctypes.c_uint32 * 4)()
    lib.density_b200_cheetah_decode_rounds(r4)
    out = d_out.cpu().numpy()
    res[name] = {"rc": rc, "size": int(d_sz.item()), "exact": int(d_sz.item()) == data.size and bool((out[:data.size] == data).all()),
                 "canary": bool((out[data.size:] == 0xA5).all()), "rounds": list(r4)}
data = np.load(f"{d}/cl33.npy")
d_in = torch.from_numpy(data).cuda()
for alg in ("cheetah", "lion"):
    want = np.load(f"{d}/cl33.{alg}.npy")
    cap = density_b200.CODECS[alg].safe_encode_buffer_size(data.size)
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_encode_device_path(density_b200.codec.ALG_IDS[alg], d_in.data_ptr(), data.size, d_out.data_ptr(), cap,
                                             d_sz.data_ptr(), st, 1)
    torch.cuda.synchronize()
    n = int(d_sz.item())
    res["encode_" + alg] = {"rc": rc, "exact": n == want.size and bool((d_out[:n].cpu().numpy() == want).all())}
print(json.dumps(res))
"""


@pytest.mark.parametrize("dec_k,enc_k", [(1, 1), (2, 3), (None, 5)])
def test_runs_per_sm_knobs(torch_cuda, sms, model, tmp_path, dec_k, enc_k):
    """DENSITY_B200_DEC_RUNS_PER_SM changes the decoder's run count (read once per process, so each value runs in a process of its own):
    the output stays exact and the rounds equal the model's at that run count, on text and on a 33 MiB corpus planted at the seams of that
    run count. DENSITY_B200_RUNS_PER_SM leaves the Cheetah and Lion streams of the run-parallel encoders bit-exact. Every value is one
    at which the SM cap binds, so the run count differs from the default's (planted.chee_runs mirrors the encoders' cap)."""
    cl33 = planted.corpus("cl33")[0]
    assert len(planted.chee_runs(cl33.size, sms, enc_k)) < len(planted.chee_runs(cl33.size, sms))
    np.save(tmp_path / "cl33.npy", cl33)
    for alg in ("cheetah", "lion"):
        np.save(tmp_path / f"cl33.{alg}.npy", oracle.encode(alg, cl33))
    cases = {}
    if dec_k is not None:
        cases["planted33k"] = cds.cl_decode_corpus(33 * MIB + 66, 5, num_sms=sms, per_sm=dec_k)[:2]
        cases["text33"] = case("text33", sms)
        for name, (data, enc) in cases.items():
            assert cds.pick_runs(enc.size, sms, dec_k) < cds.pick_runs(enc.size, sms), name
            np.save(tmp_path / f"{name}.npy", data)
            np.save(tmp_path / f"{name}.enc.npy", enc)
    (tmp_path / "child.py").write_text(_CHILD)
    env = dict(os.environ, DENSITY_B200_RUNS_PER_SM=str(enc_k),
               PYTHONPATH=os.pathsep.join([os.path.dirname(HERE), os.environ.get("PYTHONPATH", "")]))
    if dec_k is not None:
        env["DENSITY_B200_DEC_RUNS_PER_SM"] = str(dec_k)
    p = subprocess.run([sys.executable, str(tmp_path / "child.py"), str(tmp_path), "1" if cases else "0"], env=env,
                       cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    for name, (data, enc) in cases.items():
        st = model_stats(model, name + str(dec_k), sms, data, enc, per_sm=dec_k)
        r = res[name]
        print(f"DEC_RUNS_PER_SM={dec_k} {name}: {cds.pick_runs(enc.size, sms, dec_k)} runs, GPU {r['rounds'][:3]}, "
              f"model rounds {st['rounds']} settled {st['settled']} queued {st['queued']}")
        assert r["rc"] == 0 and r["canary"], (dec_k, name, r)
        assert r["rounds"][:3] == [st["rounds"], st["settled"], st["queued"]], (dec_k, name, r, st)
        if st["settled"]:
            assert st["exact"] and r["exact"], (dec_k, name, r)
        else:
            assert r["size"] == 0, (dec_k, name, r)
    for alg in ("cheetah", "lion"):
        assert res["encode_" + alg] == {"rc": 0, "exact": True}, (enc_k, alg)
