"""The generated CUDA C of every shipped machine's AIR kernels, pinned byte for byte without a GPU.

The cubins build.py ships, their cache keys and the kernel timings under profiles/ all belong to these exact sources.  One SHA-256 per
machine covers, for every component and every kernel kind (constraints, LogUp program, constraints on D2, constraint check, table-multiplicity
count), whether the library specialises it and the source it generates.  A digest that changes means the generator changed what it emits:
the shipped cubins must be rebuilt and the measured numbers no longer apply."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import build as B
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.keccak import KeccakMachine
from nexus_zkvm_b200.nexus_v1 import NexusV1Machine

u32p = C.POINTER(C.c_uint32)

DIGESTS = {
    "add-20-21-0": "be1008bc976eb01c786de907cbba232a2548001855b7af2a9f05cd9514cd9e65",
    "add-22-21-0": "aa348a8c0e7581adb175df2f8108b73faba11ae870104b2aa10a39e2bfbd442d",
    "add-16-21-0": "d87ef00749b4a2f514d69cdabf86cb30ff61b6f55ea7d14d33ce61ea66e6625d",
    "add-8-1-0": "73416475a048978aa673af1749d962b6d1b2b6ad0a91d1702f5e45374407445f",
    "add-8-2-0": "e64b2d5bf1796af98792164e75820d014bf382f6d0163ed4a0e87a475859665f",
    "add-8-2-1": "4c3b27acc6111aebc2a7fc0d384c9644873ceb4721a67371b3d99f75b637dfb9",
    "add-8-3-0": "f31ecf63be049c31f2aa16275e046c40494e2a2320adc90b305d30189c893988",
    "add-9-1-0": "0ec6c09217d28c27809c67537b4e1bbc03a978a1f871010dd925cb5fcb578e88",
    "add-9-2-0": "ce8d35235bb16cfddaebeb76b9273e1e9366b0575bc9016b54cafca2e4f80aa0",
    "add-9-2-1": "711d90f11b7e5b3eb84c4878c4a08de41a2926ceeeeb2c56fa732dc87a0aa8b9",
    "add-10-1-0": "89f7ddcb775554d24d6bf78bfdd1dca9a7b73dc99264c4c9f83d8704528444d2",
    "add-12-3-0": "d9f0bf63eddb954728e8f0dd640f2c9802374051cd6b62057525ecacd5d12a82",
    "add-16-1-0": "5cd448d7e5e4e0c41a9e8b1a588274f524cc8de1b5a8acf342b5c9e4883c3deb",
    "add-17-1-0": "9c9311ad69a7f17926d663a1ba46b65fbf080663fddbbfaeba3de01b4229d5e9",
    "add-18-1-0": "534693034afc2e9823ac6a2f2030b342982ee5d9e7b2932454313b32568a4057",
    "add-19-1-0": "c2af01b5fca0156753b18fe4850680ae66b22c261e2475d6a895102e57e5a465",
    "add-20-1-0": "72e3cc98c69ed1e86ee79f0e00142268df847d28530478596bfe749245a7b029",
    "add-21-1-0": "7921174d9e933db885de3c8d3ce49a0b31478671c6eaca6061874f7db215f891",
    "add-22-1-0": "8cd5255b55cc8341ee379d83dd71a9061ad566fa2febb7ab6e4b512b1e78ba22",
    "multi-4-11": "52467692a57efe052fc3c56f5496b3572c9ee16152e4fa7d125ec6900e567172",
    "multi-4-17": "cb89d679e1645228c588bfcc3eb2be2fa04cdf6166a3142c50e20be254a2774b",
    "multi-4-21": "df61ff340de1da300118342400ef5cac78b9fe0aa54d068ad52a4e7f34fdd8df",
    "nexus_v1-8": "f9f5a4332fbe06d578408f4ca6d9adc2c397d2c35b7f134d3f816777b5012481",
    "nexus_v1-9": "b9686c1006c20167a6eed64022d73cf7514f6cd69236f5a33c2280fb7a9b6ab4",
    "nexus_v1-12": "05452f07660314ef183664f71cfd9b406b1e42616fab29ebe6ce8d83b742d92e",
    "nexus_v1-16": "28db023156db33788fa89dcd96c6235bd4620a32dd0d1471fb8945354648b904",
    "nexus_v1-18": "303fc11c80c858477e7c8c61705b644aedfb86fc52b09b803e5d99c7686592ba",
    "nexus_v1-20": "fdedfe444f1fd7794320a740750b10d9210f95c340b59c244dc6b5e6eed51b2d",
    "nexus_v1-22": "fabac2569e0e35b58e4c3627ee97803ddcd000393135bbd38f6f9171e06c8313",
    "nexus_v1-24": "bfe1565ebc2610570e9d1aa62d4999532b7c95f98c45304302f5f98f2338fa39",
    "keccak-6": "680d796557a34bae074cc7109829df7f25e113c618fac386ce50a4bff431a670",
    "keccak-8": "f4bbca44db6acec7568fc8b7880a8d950739a35f7866cc7a73e04a1fa6011caf",
    "keccak-14": "0b391787149e7fafba861bff5661955f1ade2ce61dc9b56498aef8402777a7c5",
}


def shipped():
    out = [(f"add-{ls}-{lanes}-{int(pairs)}", lambda ls=ls, lanes=lanes, pairs=pairs: M.AddMachine(log_size=ls, n_lanes=lanes, logup_in_pairs=pairs))
           for ls, lanes, pairs in B.SHIPPED_MACHINES]
    out += [(f"multi-{s[0]}-{s[-1]}", lambda s=s: M.MultiMachine(s)) for s in B.SHIPPED_MULTI]
    out += [(f"nexus_v1-{ls}", lambda ls=ls: NexusV1Machine(ls)) for ls in B.SHIPPED_NEXUS_V1]
    out += [(f"keccak-{lp}", lambda lp=lp: KeccakMachine(lp)) for lp in B.SHIPPED_KECCAK]
    return out


def sources_digest(words):
    """SHA-256 over (component, kind, status, source) for kinds 0-3 of nb200_air_kernel_source and the count kernel (kind 4)."""
    L = nb.lib()
    w = np.ascontiguousarray(words, dtype=np.uint32)
    air = C.c_void_p()
    assert L.nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(air)) == 0
    h = hashlib.sha256()
    try:
        for comp in range(L.nb200_air_n_components(air)):
            for kind in range(5):
                p = C.c_void_p()
                if kind < 4:
                    st = L.nb200_air_kernel_source(air, C.c_uint32(comp), C.c_int(kind), C.byref(p))
                else:
                    st = L.nb200_air_count_kernel_source(air, C.c_uint32(comp), C.byref(p))
                src = b""
                if st == 0:
                    src = C.string_at(p)
                    L.nb200_free(p)
                h.update(b"%d:%d:%d:%d:" % (comp, kind, st, len(src)) + src)
    finally:
        L.nb200_air_free(air)
    return h.hexdigest()


@pytest.mark.parametrize("name,make", shipped(), ids=[n for n, _m in shipped()])
def test_shipped_kernel_sources_are_pinned(name, make):
    assert sources_digest(make().words) == DIGESTS[name]


def test_every_shipped_machine_is_pinned():
    assert sorted(DIGESTS) == sorted(n for n, _m in shipped())
