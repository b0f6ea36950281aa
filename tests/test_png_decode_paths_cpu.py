"""CPU: every refusal site of the device PNG decoder's inflate (csrc/png_inflate.cu) is reached by a stream, and the
decoder's tables and PIL's nearest index hold at the edges.

* Each `return fail(...)` / `return P3D_PNG_E...` of the source is listed in SITES against the malformed streams that
  reach it (tests/png_oracle.py: malformed_streams and refusal_streams), or in DEVICE_SITES against the GPU test that
  reaches it.  A new site without an entry fails here.
* Reaching is checked, not assumed: a copy of png_inflate.cu whose every site returns its own code (100 + its index) is
  built next to the tree's objects, and p3d_png_inflate_host, the inflate the kernel runs, must return exactly the code of
  the listed site for each listed stream.  The real build must return the stream's P3D_PNG_* status, and Python's zlib
  must refuse the stream or inflate it to a length other than the image's.
* The device (`c_*`) and host (`h_*`) copies of the length and distance tables are equal, and equal RFC 1951's.
* png_oracle.nearest_index equals PIL's nearest resize at outputs up to 32,768 and awkward inputs; the "-1 past the
  edge" branch of nearest_table cannot be reached inside the decoder's envelope (argument and check below)."""
import os
import re
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

from tests import png_oracle as po

# anchor -> the streams that reach its site.  An anchor is one or more consecutive source lines (each given by a piece of
# it, '\n' between lines) that occurs once; its last line holds the site.
SITES = {
    # dynamic_header
    'hlit > 286 || hdist > 30': ['hlit_287', 'hdist_31'],
    'cl[P3D_TAB(clorder)[i]] = (uint8_t)br.bits(3);\n}\nif (br.past_end())': ['truncated_in_code_length_lengths'],
    'if (!build(t.cl,': ['oversubscribed_code_length_code'],
    'const int s = decode(br, t.cl, t.clfast, 7);\nif (br.past_end())': ['truncated_in_code_lengths'],
    'if (s < 0) return P3D_PNG_ECODES;': ['code_length_symbol_outside_the_code'],
    'if (i == 0) return P3D_PNG_ECODES;': ['repeat_16_first'],
    'rep = s == 17 ?\n}\nif (br.past_end())': ['truncated_in_repeat_bits'],
    'if (i + rep > hlit + hdist)': ['repeat_past_hlit_hdist'],
    'if (t.lens[256] == 0)': ['no_end_of_block_code'],
    'if (!build(t.lit,': ['incomplete_literal_code'],
    'if (!build(t.dist,': ['oversubscribed_distance_code'],
    # run: zlib header and trailer
    'flg = br.bits(8);\nif (br.past_end())': ['empty_stream'],
    '(flg & 32)) return fail': ['bad_fcheck', 'cinfo_8', 'method_7', 'preset_dictionary'],
    'a = a << 8 | br.bits(8);\nif (br.past_end())': ['truncated_adler'],
    'if (p != out_len)': ['too_short'],
    # run: block headers and stored blocks
    'const int type = (int)br.bits(2);\nif (br.past_end())': ['truncated_after_the_zlib_header'],
    'nlen = br.bits(16);\nif (br.past_end())': ['truncated_in_stored_len_nlen'],
    '(len ^ 0xffffu) != nlen': ['stored_nlen'],
    'if (len > br.n - q)': ['stored_len_past_the_input'],
    'if (len > br.n - q)\nif (len > out_len - p)': ['too_long_by_a_stored_block'],
    'if (type == 3)': ['block_type_3'],
    # run: Huffman blocks
    'const int s = decode(br, t.lit, t.lfast, kLitFast);\nif (br.past_end())': ['truncated_mid_block'],
    'if (s < 0) return fail(P3D_PNG_ESYMBOL);': ['literal_bits_outside_a_one_code_code'],
    'if (p >= out_len)': ['too_long'],
    'if (s > 285)': ['literal_286'],
    'const int ds = decode(br, t.dist, t.dfast, kDistFast);\nif (br.past_end())': ['truncated_before_a_distance_code'],
    'if (ds < 0 || ds > 29)': ['match_without_distance_codes', 'fixed_distance_symbol_30', 'fixed_distance_symbol_31'],
    'P3D_TAB(dext)[ds]);\nif (br.past_end())': ['truncated_in_distance_extra_bits'],
    'if (dist > p)': ['distance_past_start'],
    'if (dist > p)\nif (len > out_len - p)': ['too_long_by_a_match'],
}
# sites the host inflate never runs: check_job guards the kernel's job table, and tests/test_png_decode_paths_gpu.py's
# test_refused_jobs_fail_alone hands the kernel one job per line
DEVICE_SITES = {
    'if (!need || j.slot < 0': 'channels 2',
    'if (j.in_offset > b.in_bytes': 'input span past the buffer',
    '(j.ws_offset & 15)': 'workspace offset not 16-byte aligned',
}
# `return fail(e)` hands dynamic_header's code on: each dynamic_header site above goes through it
FORWARDS = {'if (e) return fail(e);'}

SITE_RE = re.compile(r'return (?:fail\((P3D_PNG_E\w+|e)\)|(P3D_PNG_E\w+));')


def source():
    from panic3d_b200 import _build
    return open(os.path.join(_build.CSRC, 'png_inflate.cu')).read()


def site_lines(text):
    """Indices of the source lines that hold a refusal site (one per line)."""
    lines = text.splitlines()
    res = []
    for i, ln in enumerate(lines):
        k = len(SITE_RE.findall(ln))
        assert k <= 1, f'two sites on line {i + 1}'
        if k:
            res.append(i)
    return res


def locate(text, anchor):
    lines = text.splitlines()
    parts = anchor.split('\n')
    hits = [i for i in range(len(lines) - len(parts) + 1) if all(p in lines[i + j] for j, p in enumerate(parts))]
    assert len(hits) == 1, f'anchor {anchor!r} found {len(hits)} times'
    return hits[0] + len(parts) - 1


def all_streams():
    res = {k: (s, n, c) for k, (s, n, c) in po.malformed_streams().items()}
    res.update(po.refusal_streams())
    return res


@pytest.fixture(scope='module')
def L():
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _lib, imageio  # noqa: F401  (register the p3d_png_* prototypes)
    return _lib.lib()


def inflate(lib, stream, n):
    raw = np.zeros(n, np.uint8)
    s = np.frombuffer(stream, np.uint8)
    return lib.p3d_png_inflate_host(s.ctypes.data if s.size else None, s.size, raw.ctypes.data, n)


@pytest.fixture(scope='module')
def site_lib(L):
    """The library with png_inflate.cu's site k returning 100 + k, built in a temporary directory."""
    import ctypes as C
    import shutil
    from panic3d_b200 import _build
    text = source()
    lines = text.splitlines(keepends=True)
    for k, i in enumerate(site_lines(text)):
        lines[i] = SITE_RE.sub(lambda m: m.group(0) if m.group(1) == 'e' else
                               (f'return fail({100 + k});' if m.group(1) else f'return {100 + k};'), lines[i])
    with tempfile.TemporaryDirectory() as d:
        csrc = os.path.join(d, 'csrc')
        shutil.copytree(_build.CSRC, csrc)
        open(os.path.join(csrc, 'png_inflate.cu'), 'w').write(''.join(lines))
        nvcc = _build.find_nvcc()
        src = os.path.join(_build.CSRC, 'png_inflate.cu')
        obj, lib = os.path.join(d, 'png_inflate.o'), os.path.join(d, 'libsites.so')
        objs = [obj if s == src else _build.object_path(s) for s in _build.sources()]
        for cmd in (_build.compile_cmd(nvcc, os.path.join(csrc, 'png_inflate.cu'), obj, ['-I', _build.CSRC]),
                    _build.link_cmd(nvcc, lib, objs)):
            r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            assert r.returncode == 0, r.stdout
        h = C.CDLL(lib)
        h.p3d_png_inflate_host.restype = C.c_int
        h.p3d_png_inflate_host.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        yield h


def test_every_refusal_site_is_listed():
    text = source()
    sites = site_lines(text)
    listed = {}
    for anchor in list(SITES) + list(DEVICE_SITES) + list(FORWARDS):
        i = locate(text, anchor)
        assert i in sites, f'{anchor!r} does not end on a refusal site'
        assert i not in listed, f'line {i + 1} listed twice: {listed.get(i)!r} and {anchor!r}'
        listed[i] = anchor
    missing = [f'{i + 1}: {text.splitlines()[i].strip()}' for i in sites if i not in listed]
    assert not missing, 'refusal sites without a stream:\n' + '\n'.join(missing)
    names = all_streams()
    for anchor, streams in SITES.items():
        assert streams and all(s in names for s in streams), anchor
    gpu = open(os.path.join(os.path.dirname(__file__), 'test_png_decode_paths_gpu.py')).read()
    assert 'def test_refused_jobs_fail_alone' in gpu and all(why in gpu for why in DEVICE_SITES.values())


def test_each_stream_reaches_its_site(site_lib):
    text = source()
    index = {i: k for k, i in enumerate(site_lines(text))}
    streams = all_streams()
    for anchor, names in SITES.items():
        want = 100 + index[locate(text, anchor)]
        for name in names:
            stream, n, _ = streams[name]
            got = inflate(site_lib, stream, n)
            assert got == want, (name, anchor, got, want)


@pytest.mark.parametrize('name', list(po.refusal_streams()))
def test_refusal_streams_get_their_status_and_zlib_agrees(L, name):
    from panic3d_b200 import imageio as pio
    stream, n, code = po.refusal_streams()[name]
    rc = inflate(L, stream, n)
    assert rc == code, (name, rc, pio.PNG_STATUS.get(rc))
    try:
        out = zlib.decompressobj().decompress(stream)
    except zlib.error:
        return
    assert len(out) != n, name


@pytest.mark.parametrize('name', list(po.path_streams()))
def test_path_streams_inflate_on_the_host(L, name):
    h, w, c, depth, stream, raw = po.path_streams()[name]
    assert zlib.decompress(stream) == raw and len(raw) == h * (1 + w * c * depth // 8)
    out = np.zeros(len(raw), np.uint8)
    s = np.frombuffer(stream, np.uint8)
    assert L.p3d_png_inflate_host(s.ctypes.data, s.size, out.ctypes.data, len(raw)) == 0
    assert out.tobytes() == raw


def test_path_streams_take_the_paths_they_name():
    """The streams zlib never writes are what their names say: read their block types and dynamic headers back."""
    streams = po.path_streams()
    blocks = read_blocks(streams['dynamic_fixed_fixed_dynamic_stored_fixed'][4])
    assert [b['type'] for b in blocks] == [2, 1, 1, 2, 0, 1]
    hdr = read_blocks(streams['hlit_286_hdist_30_15_bit_codes'][4])[0]
    assert (hdr['hlit'], hdr['hdist']) == (286, 30)
    assert hdr['lens'][7] == hdr['lens'][270] == 15 and hdr['lens'][286 + 2] == hdr['lens'][286 + 29] == 15
    assert (16, 6) in read_blocks(streams['repeat_16_across_the_two_lists'][4])[0]['clsyms']
    syms = read_blocks(streams['repeat_18_of_138'][4])[0]['clsyms']
    assert (18, 138) in syms


def read_blocks(stream):
    """A minimal walk of a zlib stream's blocks: the type of each, and for dynamic blocks hlit, hdist, the code-length
    symbols (repeats as (symbol, count)) and the lengths.  Symbols are decoded bit by bit and dropped."""
    bits = np.unpackbits(np.frombuffer(stream[2:], np.uint8), bitorder='little')
    pos = 0

    def get(k):
        nonlocal pos
        v = int(sum(int(b) << i for i, b in enumerate(bits[pos:pos + k])))
        pos += k
        return v

    def huff_decode(lens):
        codes = po.canonical(lens)
        table = {(l, c): s for s, (l, c) in enumerate(zip(lens, codes)) if l}
        code, l = 0, 0
        while True:
            code = code << 1 | get(1)
            l += 1
            if (l, code) in table:
                return table[(l, code)]

    res = []
    while True:
        final, typ = get(1), get(2)
        blk = {'type': typ}
        res.append(blk)
        if typ == 0:
            pos = (pos + 7) // 8 * 8
            n = get(16)
            get(16)
            pos += 8 * n
        else:
            if typ == 1:
                ll, dl = po.FIXED_LIT, [5] * 32
            else:
                hlit, hdist, hclen = get(5) + 257, get(5) + 1, get(4) + 4
                cl = [0] * 19
                for i in range(hclen):
                    cl[po.CLORDER[i]] = get(3)
                lens, syms = [], []
                while len(lens) < hlit + hdist:
                    s = huff_decode(cl)
                    if s < 16:
                        lens.append(s)
                        syms.append(s)
                        continue
                    rep = 3 + get(2) if s == 16 else 3 + get(3) if s == 17 else 11 + get(7)
                    lens += [lens[-1] if s == 16 else 0] * rep
                    syms.append((s, rep))
                blk.update(hlit=hlit, hdist=hdist, lens=lens, clsyms=syms)
                ll, dl = lens[:hlit], lens[hlit:]
            while True:                                        # skip the block's symbols
                s = huff_decode(ll)
                if s == 256:
                    break
                if s > 256:
                    get(po.LEXT[s - 257])
                    get(po.DEXT[huff_decode(dl)])
        if final:
            return res


def c_table(text, prefix, name):
    m = re.search(prefix + name + r'\[\d+\] = \{([^}]*)\};', text)
    assert m, prefix + name
    return [int(v) for v in m.group(1).split(',')]


@pytest.mark.parametrize('name,want', [('lbase', po.LBASE), ('lext', po.LEXT), ('dbase', po.DBASE), ('dext', po.DEXT),
                                       ('clorder', po.CLORDER)])
def test_device_and_host_tables_are_equal(name, want):
    text = source()
    assert c_table(text, 'c_', name) == c_table(text, 'h_', name) == want


def test_nearest_index_against_pil_at_large_and_awkward_sizes():
    from PIL import Image
    for n_in in (1, 3, 7, 1000, 4097, 32767):
        for n_out in (1, 2, 999, 1001, 4096, 4098, 20000, 30000, 32767, 32768):
            im = Image.fromarray(np.arange(n_in, dtype=np.int32)[None], mode='I').resize((n_out, 1), Image.NEAREST)
            assert np.array_equal(np.asarray(im)[0], po.nearest_index(n_in, n_out)), (n_in, n_out)


def test_nearest_table_never_reaches_past_the_edge():
    """nearest_table's `-1` (a source index at or past n_in) is unreachable inside the envelope: the accumulated x_o =
    scale (o + 1/2) + e with |e| <= (o + 1) ulp(n_in) < n_out n_in 2^-52, and reaching n_in needs e >= scale / 2 =
    n_in / (2 n_out), i.e. n_out^2 >= 2^51, while n_out <= 32768 = 2^15.  x starts at scale / 2 > 0 and grows, so the
    `x < 0` branch is unreachable too.  Checked with the same sequential double sums at the sizes the error grows with."""
    for n_in in (1, 2, 3, 1000, 4097, 32767, 1 << 20, (1 << 28) - 1):
        for n_out in (1, 3, 1000, 4097, 30000, 32767, 32768):
            scale = n_in / n_out
            x = np.add.accumulate(np.concatenate([[scale * 0.5], np.full(n_out - 1, scale)]))
            assert x[0] > 0 and int(x[-1]) < n_in, (n_in, n_out)
    assert np.array_equal(np.add.accumulate(np.concatenate([[4097 / 32768 * 0.5], np.full(32767, 4097 / 32768)])).astype(np.int64),
                          po.nearest_index(4097, 32768))
