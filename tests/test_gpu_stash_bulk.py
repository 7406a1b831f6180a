"""The fp32 training stash of the tensor-core engine, byte for byte: tc_field_fwd writes h0..h7, feat, hr, enc, denc and the ReLU gate
bits, tc_dgrad writes dy0..dy7, dfeat, dyr and dyc.  Each region is hashed in place (all Mpad rows, padding rows included) after
nnb_render_fwd and again after nnb_render_bwd, and compared with SHA-256 digests recorded from the build whose epilogues stored the stash
straight from registers.  How the bytes reach global memory may change; the bytes may not.

Cases: D = 64, 128 and 256 at the C2 shape (1024 rays x 128 samples), a ragged M (301 x 17 = 5117, not a multiple of 128), 16 and 1024
samples per ray, and a 2-ray call (one partial tile).

Recording (on a GPU, with the library to take the digests from):  python tests/test_gpu_stash_bulk.py"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import nerf_oracle as O  # noqa: E402
from test_gpu_relu_mask import _render, layout  # noqa: E402

CASES = [(256, 1024, 128), (128, 1024, 128), (64, 1024, 128), (256, 301, 17), (128, 333, 16), (64, 9, 1024), (256, 2, 17)]
FWD = ["h%d" % l for l in range(8)] + ["feat", "hr", "enc", "denc", "gates"]
BWD = ["dy%d" % l for l in range(8)] + ["dfeat", "dyr", "dyc"]


def _regions(lay):
    """name -> (byte offset, bytes) of every stash region of the layout"""
    Mp, D = lay["Mpad"], lay["D"]
    r = {"h%d" % l: (lay["h"][l], Mp * D * 4) for l in range(8)}
    r.update(feat=(lay["feat"], Mp * D * 4), hr=(lay["hr"], Mp * D * 2), enc=(lay["enc"], Mp * 64 * 4), denc=(lay["denc"], Mp * 32 * 4),
             gates=(lay["gates"], Mp * D + Mp * D // 16))
    r.update({"dy%d" % l: (lay["dy"][l], Mp * D * 4) for l in range(8)})
    r.update(dfeat=(lay["dfeat"], Mp * D * 4), dyr=(lay["dyr"], Mp * D * 2), dyc=(lay["dyc"], Mp * 16))
    return r


def _hash(ws, regs, names):
    torch.cuda.synchronize()
    return {n: hashlib.sha256(ws[regs[n][0]:regs[n][0] + regs[n][1]].cpu().numpy().tobytes()).hexdigest()[:16] for n in names}


def digests(D, N, S):
    """(forward regions after nnb_render_fwd, every region after nnb_render_bwd)"""
    from nope_nerf_b200 import _lib as L
    call = _render(O.init_params(seed=5, D=D), D, N, S, seed=11)
    ws, lay = call.ws, layout(N, S, D)
    regs = _regions(lay)
    fwd = _hash(ws, regs, FWD)
    rng = np.random.default_rng(7)
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    g_rgb = cu(rng.normal(0, 1, (N, 3)).astype(np.float32))
    g_dp = cu(rng.normal(0, 1, N).astype(np.float32)); g_dg = cu(rng.normal(0, 1, N).astype(np.float32))
    g_w = torch.zeros(L.num_params(D), device="cuda")
    call.backward(g_rgb, g_dp, g_dg, g_w, torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4, device="cuda"), None,
                  torch.zeros(2, device="cuda"))   # hands the workspace back to the pool; ws stays alive
    return fwd, _hash(ws, regs, FWD + BWD)


# recorded from the register-store build (H100 80GB HBM3, 700 W)
DIGESTS = {
    "256_1024_128": {
        "h0": "31c8971033d60696", "h1": "0fbf63d8b32acc5e", "h2": "d6c1a7170e12d813", "h3": "08c39a2a56c10d63",
        "h4": "3be8e222fbab02cb", "h5": "ed0fb3e475d149a4", "h6": "9c586bc04fcc22b3", "h7": "f65d74e70bcee925",
        "feat": "e9f9e733bf9e4f98", "hr": "cf5c249cabb918ce", "enc": "a80f835eba526e22", "denc": "702ce5b003fe688c",
        "gates": "956305b2db61d67d", "dy0": "eda61189989b5ec9", "dy1": "ccdf23691988e71e", "dy2": "828b7b5f02a510d3",
        "dy3": "58db3410cd6bccac", "dy4": "8627e41fd3450a4a", "dy5": "f1e523eea9ee2ad6", "dy6": "81072d406374844c",
        "dy7": "34bc11824aa55d5f", "dfeat": "c726a874d9520519", "dyr": "fd7bbeb4f50f5780", "dyc": "e5fe5a50cbc124da",
    },
    "128_1024_128": {
        "h0": "25e6a20c5ece7ee2", "h1": "b1b45124fec5ff55", "h2": "5dbfe1c62a196f0e", "h3": "5cf13197bbc5567e",
        "h4": "5aee5689f413a58c", "h5": "ec52d489498ceb42", "h6": "8e5b50b8ff2c3e0a", "h7": "d45af2829efd368c",
        "feat": "08139413ad0d8120", "hr": "8c93909502f9d272", "enc": "a80f835eba526e22", "denc": "702ce5b003fe688c",
        "gates": "daddfd18464a0d1d", "dy0": "716cfbdaa40461e2", "dy1": "c82f874b42d3370a", "dy2": "82c4a28771f02e34",
        "dy3": "fa1e1c17f3cedc8e", "dy4": "6cafc9714bf8dc50", "dy5": "c7a5561c0ed920a6", "dy6": "bdb07e0700266875",
        "dy7": "27ea184d499af4d9", "dfeat": "9c4eb1e74f50f799", "dyr": "db6f5339ff386ea4", "dyc": "ea6948f64fadb6a0",
    },
    "64_1024_128": {
        "h0": "79b52d2ceb7f8f20", "h1": "22423d80b88333aa", "h2": "f16f80a6c4499cd3", "h3": "163b9d498203a021",
        "h4": "df1c3f1a94688b20", "h5": "96a8b70e47eea401", "h6": "09c6ba5458358fd3", "h7": "74e928e0e3166c48",
        "feat": "74ea6676af7ab0d3", "hr": "358eb3c1ef6c9f3c", "enc": "a80f835eba526e22", "denc": "702ce5b003fe688c",
        "gates": "f0fff9703a83b295", "dy0": "f6681a879859f50f", "dy1": "713ca62cbe892bdb", "dy2": "c645c887aff54ba3",
        "dy3": "9652ce66e70a3aa2", "dy4": "24e17b175f9a497e", "dy5": "f7b4e15114d00090", "dy6": "80f0b18e13efffb5",
        "dy7": "3e6c4b42cfd5d4b7", "dfeat": "a7adf4a538ec6855", "dyr": "c74b2ec14f2fcc6f", "dyc": "a5971fe292d7d01e",
    },
    "256_301_17": {
        "h0": "64b2780731da14f5", "h1": "4484c9d7616ce00f", "h2": "dc60e97c0369bc57", "h3": "c189d28b405d7582",
        "h4": "688dbb1a822bb23a", "h5": "2fc34ab89c0252c1", "h6": "7bbe882f17d1df31", "h7": "b2ad4adad85ccfe4",
        "feat": "a58861d3b7043417", "hr": "668897d3bb91d981", "enc": "6a7883e047aedade", "denc": "1e17b48e09fca550",
        "gates": "a7878f2cb9fee68a", "dy0": "6c1b46b90e2bbce4", "dy1": "c5869b059be1dcc5", "dy2": "fedaf53b18edf1c4",
        "dy3": "4cc36d7eea399a57", "dy4": "21f10986a9d155b6", "dy5": "0b9c8c6eaaaac926", "dy6": "6f0457412b9df7be",
        "dy7": "777cb572ec4bc947", "dfeat": "2729198e0ec6c518", "dyr": "23fa8f22307d6bf9", "dyc": "1be2a3190169b65a",
    },
    "128_333_16": {
        "h0": "ef031016a13ea09e", "h1": "e58b7ebe55ceb896", "h2": "1b8aeaec0f3909c1", "h3": "17ab5ee18636fa9b",
        "h4": "54d6a546a3d7ca4a", "h5": "7a8b4caa2892eb04", "h6": "28f056ae95c628d0", "h7": "51048f550ef41252",
        "feat": "f6f555c6444986a7", "hr": "9b50129f6f63bc6d", "enc": "f95a1dc0c8e1f7bf", "denc": "feb9e10f73db0637",
        "gates": "cee1ca27c7249aff", "dy0": "596c94c725664dc1", "dy1": "d1c408d8f6ee0f68", "dy2": "27f2bc9adb6a7289",
        "dy3": "98952858624159be", "dy4": "bd79dafe4b381436", "dy5": "e3d7075fcf58eab6", "dy6": "5a36e2ab1ee53afd",
        "dy7": "226001a6577bad0c", "dfeat": "6fffcfeeb8add187", "dyr": "734d1bd35e87ba42", "dyc": "3e7863c9cbfc48f1",
    },
    "64_9_1024": {
        "h0": "732f12690af7e422", "h1": "7166cfb6e2b00e2c", "h2": "3b32d5adc2cd0f78", "h3": "276e9c15d4d6d432",
        "h4": "ca87a128bf54ca4b", "h5": "81c4995919b5e787", "h6": "03227cac12256ea4", "h7": "8f54ade718c1270f",
        "feat": "3ee65ae1ed06b587", "hr": "fc7dc1d6f9efbd1b", "enc": "426603a4260e4761", "denc": "da357c0075a6848c",
        "gates": "654a7b70281ef948", "dy0": "ed8802e38ceb6589", "dy1": "7f7ba9f101db4285", "dy2": "2e52c6dc16957261",
        "dy3": "36d3a5a4929c99d7", "dy4": "0c1584f14dc042fc", "dy5": "561bedda12d41f58", "dy6": "c7f0ef2aabcbd0c6",
        "dy7": "ccbb76cd55d2e6ea", "dfeat": "8e656bd4c3ddb2f4", "dyr": "2dd2ab1dca5c4a78", "dyc": "a5ea4974e7355172",
    },
    "256_2_17": {
        "h0": "7b7b277bb1a4839d", "h1": "e009050d29c84912", "h2": "ad9e7f7df87fff26", "h3": "19a97a8f133f2606",
        "h4": "843526d8a91162d4", "h5": "282f9462449cc6d7", "h6": "e1ad540563bbdad2", "h7": "b5cff9ebad8865a9",
        "feat": "db7278bc7cf74cbf", "hr": "6909df34b3d08ad9", "enc": "e43e0aabe428d826", "denc": "e5c38728670af558",
        "gates": "18c9d86c4bd532ee", "dy0": "9bfb3f175c29aec7", "dy1": "e3a2baf71a54d310", "dy2": "d08ab21331e793ba",
        "dy3": "d0c74d9775236070", "dy4": "43ae490c4e143b3e", "dy5": "3e86c00acd446c07", "dy6": "5d3bb13328c19e53",
        "dy7": "f1609b2df34104cb", "dfeat": "8f034806992f0287", "dyr": "c058b59cbd3c261f", "dyc": "a24b32a484479246",
    },
}


@pytest.mark.gpu
@pytest.mark.parametrize("D,N,S", CASES)
def test_stash_bytes_unchanged(D, N, S):
    key = "%d_%d_%d" % (D, N, S)
    fwd, bwd = digests(D, N, S)
    want = DIGESTS[key]
    assert {n: fwd[n] for n in FWD} == {n: want[n] for n in FWD}, "forward stash differs"
    assert bwd == want, "stash after the backward differs"


if __name__ == "__main__":
    out = {}
    for D, N, S in CASES:
        fwd, bwd = digests(D, N, S)
        assert all(fwd[n] == bwd[n] for n in FWD), "the backward changed a forward region"
        out["%d_%d_%d" % (D, N, S)] = bwd
    print(json.dumps(out, indent=1))
