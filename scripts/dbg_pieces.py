"""Debug aid: run the device inflate batch on a config-2 style workload and analyse the piece tables
(how much of every stream the speculative helper lanes delivered)."""
import os, sys, numpy as np, torch, collections
sys.path.insert(0, '.')
from archive_b200 import _ffi, synth
n = int(os.environ.get('N_UNITS', 4096)); UNIT = 65536
L = _ffi.ensure_init(0)
w = synth.gzip_workload(n, UNIT, stream0=0, cache_dir=os.environ.get('B200Z_CACHE', '/tmp/b200z_cache'))
blob, moff = w["blob"], w["member_off"]
hdr = 18
in_off = (moff[:-1] + hdr).astype(np.uint64); in_len = (moff[1:] - moff[:-1] - hdr).astype(np.uint32)
out_off = (np.arange(n, dtype=np.uint64) * UNIT); out_cap = np.full(n, UNIT, dtype=np.uint32)
dev = torch.device('cuda:0')
d_in = torch.empty(len(blob) + 64, dtype=torch.uint8, device=dev); d_in[:len(blob)].copy_(torch.from_numpy(blob.copy()))
d_out = torch.empty(n * UNIT, dtype=torch.uint8, device=dev)
t = lambda a, ty: torch.from_numpy(a.view(ty)).to(dev)
d_in_off, d_in_len, d_out_off, d_out_cap = t(in_off, np.int64), t(in_len, np.int32), t(out_off, np.int64), t(out_cap, np.int32)
d_ol = torch.zeros(n, dtype=torch.int32, device=dev); d_st = torch.full((n,), -99, dtype=torch.int32, device=dev); d_us = torch.zeros(n, dtype=torch.int32, device=dev)
ws_bytes = L.b200z_inflate_workspace_bytes(n, len(blob), n * UNIT)
d_ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
rc = L.b200z_inflate_batch_device(d_in.data_ptr(), d_in_off.data_ptr(), d_in_len.data_ptr(), d_out.data_ptr(), d_out_off.data_ptr(),
                                  d_out_cap.data_ptr(), d_ol.data_ptr(), d_st.data_ptr(), d_us.data_ptr(), n, d_ws.data_ptr(), ws_bytes, 0)
torch.cuda.synchronize(); assert rc == 0
# replicate inflate_ws_extent_for / inflate_ws_carve
PW, US = 2 + 3 * 30, 7 * 64 * 4
def ws_b(nu, ext):
    tok = (ext * 4 + 511) & ~255; hs = (ext >> 2) + 64; hb = (7 * hs * 4 + 255) & ~255
    return tok + hb + ((nu * PW * 4 + 255) & ~255) + ((nu * US + 255) & ~255) + 256
ext = n * UNIT  # the largest extent with ws_b(n, ext) <= ws_bytes
while ws_b(n, ext + 1) <= ws_bytes:
    ext += 1
tok = (ext * 4 + 511) & ~255; hs = (ext >> 2) + 64; hb = (7 * hs * 4 + 255) & ~255
P = d_ws[tok + hb: tok + hb + n * PW * 4].cpu().numpy().view(np.uint32).reshape(n, PW)
npc = P[:, 0]
print('status', collections.Counter(d_st.cpu().numpy().tolist()), 'pieces hist', sorted(collections.Counter(npc.tolist()).items()))
own = np.zeros(n); tot = np.zeros(n)
for u in range(n):
    for i in range(npc[u]):
        src, st, c = P[u, 2 + 3 * i: 5 + 3 * i]
        tot[u] += c
        if src == 0: own[u] += c
frac = own / tot
print('own-token share: mean %.3f  p50 %.3f  p99 %.3f  max %.3f' % (frac.mean(), np.median(frac), np.percentile(frac, 99), frac.max()))
worst = np.argsort(-frac)[:5]
for u in worst:
    print('unit', u, 'own', frac[u], [(int(P[u, 2 + 3 * i]), int(P[u, 3 + 3 * i]), int(P[u, 4 + 3 * i])) for i in range(npc[u])])
import zlib
o = d_out.cpu().numpy()
bad = sum(1 for u in range(0, n, 97) if zlib.crc32(o[u * UNIT:(u + 1) * UNIT].tobytes()) != zlib.crc32(zlib.decompress(blob[moff[u]:moff[u + 1]].tobytes(), 31)))
print('crc mismatches in sample', bad)
