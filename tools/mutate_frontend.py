#!/usr/bin/env python3
"""Mutation check of a host-side front-end's tests (dev-time; CPU only): every (old, new) pair below is applied to a copy of the
source, the copy is compiled on its own with g++, its entry points replace the library's inside a pytest run of the front-end's
tests, and a mutant that no test kills is reported.  `python tools/mutate_frontend.py aac|vorbis`."""
import ctypes
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "symphonia_b200", "csrc")

TARGETS = {
    "aac": dict(src="aac_frontend.cpp", prefix="symgpu_aac_fe_", tests=["tests/test_aac_frontend.py", "tests/test_zz_adts_aac_to_pcm.py"], mutants=[
        ("while (bs.left() > 3)", "while (bs.left() > 2)"),
        ("if (count == 255) count += bs.read(8);", "if (count == 254) count += bs.read(8);"),
        ("if (count == 15) count += bs.read(8) - 1;", "if (count == 15) count += bs.read(8);"),
        ("CHECK(l < 64);", "CHECK(l < 65);"),
        ("CHECK(cb != RESERVED_HCB);", ""),
        ("if (inc < esc) break;", "if (inc <= esc) break;"),
        ("CHECK(k + len <= max_sfb);", "CHECK(k + len < max_sfb + 2);"),
        ("int32_t scf_int = 155,", "int32_t scf_int = 156,"),
        ("int32_t(global_gain) - 90 + 100", "int32_t(global_gain) - 91 + 100"),
        ("int32_t(bs.read(9)) - 256", "int32_t(bs.read(9)) - 255"),
        ("CHECK(scf_normal >= 0 && scf_normal < 256);", "CHECK(scf_normal >= 0 && scf_normal < 255);"),
        ("CHECK(scf_noise >= 0 && scf_noise < 256);", "CHECK(scf_noise >= 1 && scf_noise < 256);"),
        ("CHECK(scf_int >= 0 && scf_int < 256);", "CHECK(scf_int >= 0 && scf_int < 257);"),
        ("CHECK(n < 9);", "CHECK(n < 10);"),
        ("const float x = a < 4 ? -T.pow43[4 - a]", "const float x = a <= 4 ? -T.pow43[4 - a]"),
        ("const uint32_t mod = cb < 9 ? 8 : 13;", "const uint32_t mod = cb < 10 ? 8 : 13;"),
        ("const uint32_t max_order = long_win ? 12 : 7;", "const uint32_t max_order = long_win ? 12 : 8;"),
        ("const uint32_t max_order = long_win ? 12 : 7;", "const uint32_t max_order = long_win ? 13 : 7;"),
        ("CHECK(t.order <= max_order);", "CHECK(t.order < max_order);"),
        ("(coef_res ? 4u : 3u) - (compress ? 1u : 0u)", "(coef_res ? 4u : 3u) - (compress ? 0u : 1u)"),
        ("CHECK(!has_pulse || long_win);", ""),
        ("if (k >= 1024) return;", "if (k > 1024) return;"),
        ("if (pulse_start >= b.len - 1) return;", "if (pulse_start >= b.len) return;"),
        ("while (b.v[band + 1] <= k) ++band;", "while (b.v[band + 1] < k) ++band;"),
        ("if (base > 0.0f) base += float(pulse_amp[i]);", "if (base >= 0.0f) base += float(pulse_amp[i]);"),
        ("if (max_sfb < max_bands) max_bands = max_sfb;", ""),
        ("CHECK(ms_mask_present != 3);", ""),
        ("const bool invert = ms_mask_present == 1 && ms_used[g][s];", "const bool invert = ms_mask_present != 0 && ms_used[g][s];"),
        ("} else if (c0 == NOISE_HCB || c1 == NOISE_HCB) {", "} else if (c0 == NOISE_HCB) {"),
        ("} else if (c0 == NOISE_HCB || c1 == NOISE_HCB) {", "} else if (c1 == NOISE_HCB) {"),
        ("if (w > 0 && !a.grouping[w - 1]) ++g;", "if (w > 0 && !a.grouping[w]) ++g;"),
        ("prev_window_sequence = seq, prev_window_shape = shape;", "prev_window_sequence = seq;"),
        ("CHECK(max_sfb + 1 <= bands().len);", "CHECK(max_sfb <= bands().len);"),
        ("(long_win ? 1u : 8u)", "8u"),
        ("CHECK((pair ? channel + 1 : channel) < channels);", "CHECK((pair ? channel + 1 : channel) <= channels);"),
        ("if (cur_ch != fe->channels) return SYMGPU_ERR_UNSUPPORTED;", ""),
        ("window_shape = prev_window_shape = false;", "prev_window_shape = false;"),
        ("                case 3: {", "                {"),
        ("u.tns_first = nf ? tns_base + total : 0;", "u.tns_first = nf ? total : 0;"),
        ("if (align) bs.realign();", ""),
        ("bs.ignore(uint64_t(count - 1) * 8);", "bs.ignore(uint64_t(count) * 8);"),
        ("float(int16_t(lcg.next() >> 16))", "float(int16_t(lcg.next() >> 15))"),
        ("if (predictor) return SYMGPU_ERR_UNSUPPORTED;", "if (predictor) return SYMGPU_ERR_DECODE;"),
        ("CHECK(!gain_control);", ""),
        ("uint32_t state = 0x1f2e3d4c;", "uint32_t state = 0x1f2e3d4d;"),
        ("if (a) sx = sign_of(bs.read(1));", "if (a > 1) sx = sign_of(bs.read(1));"),
        ("case 2: return SYMGPU_ERR_UNSUPPORTED;", "case 2: return SYMGPU_ERR_DECODE;"),
        ("CHECK(pairs[pair_no]->is_pair == pair);", ""),
        ("CHECK(pairs[pair_no]->channel == channel);", ""),
        ("2.51984209978974632953f * scale", "2.5198421f * scale * 1.0000001f"),
    ]),
    "asc": dict(src="aac_frontend.cpp", prefix="symgpu_aac_", tests=["tests/test_aac_frontend.py"], mutants=[
        ("if (v == 31) v = bs.read(6) + 32;", "if (v == 31) v = bs.read(6) + 31;"),
        ("if (idx <= 12) rate = kRates[idx];", "if (idx <= 11) rate = kRates[idx];"),
        ("else if (idx == 15) rate = bs.read(24);", "else if (idx >= 14) rate = bs.read(24);"),
        ("CHECK(out->sample_rate != 0);", ""),
        ("CHECK(idx <= 7);", "CHECK(idx <= 8);"),
        ("static const uint8_t kChannels[8] = {0, 1, 2, 3, 4, 5, 6, 8};", "static const uint8_t kChannels[8] = {0, 1, 2, 3, 4, 5, 6, 7};"),
        ("if (aot == 5 || aot == 29) {  // SBR / PS", "if (aot == 5) {  // SBR / PS"),
        ("out->ps_present = aot == 29,", "out->ps_present = 0,"),
        ("if (aot == 22 && (st = channel_config(out->ext_channels)) != SYMGPU_OK) return st;", ""),
        ("out->samples = short_frame ? 960 : 1024;", "out->samples = 1024;"),
        ("if (depends_on_core) bs.read(14);", "if (depends_on_core) bs.read(13);"),
        ("if (out->channels == 0) return SYMGPU_ERR_UNSUPPORTED;  // program config element", ""),
        ("if (aot == 6 || aot == 20) bs.read(3);", "if (aot == 6) bs.read(3);"),
        ("if (aot == 22) bs.read(5), bs.read(11);", ""),
        ("if (aot == 17 || aot == 19 || aot == 20 || aot == 23) bs.read(3);", "if (aot == 17 || aot == 19 || aot == 20) bs.read(3);"),
        ("if (extension_flag3) return SYMGPU_ERR_UNSUPPORTED;", ""),
        ("if (ep_config >= 2) return SYMGPU_ERR_UNSUPPORTED;", "if (ep_config >= 3) return SYMGPU_ERR_UNSUPPORTED;"),
        ("if (out->has_ext && bs.left() >= 16) {", "if (out->has_ext && bs.left() >= 17) {"),
        ("if (out->has_ext && bs.left() >= 16) {", "if (bs.left() >= 16) {"),
        ("if (sync == 0x2b7) {", "if (sync == 0x2b6) {"),
        ("if (bs.left() >= 12) {", "if (bs.left() >= 13) {"),
        ("if (bs.read(11) == 0x548) out->ps_present = bs.read_bool();", "if (bs.read(11) == 0x549) out->ps_present = bs.read_bool();"),
        ("if (n < 2) return SYMGPU_ERR_DECODE;", "if (n < 1) return SYMGPU_ERR_DECODE;"),
        ("if (asc.object_type != 2 || asc.sbr_present || asc.channels > 2 || asc.samples != 1024) return SYMGPU_ERR_UNSUPPORTED;", "if (asc.object_type != 2 || asc.channels > 2 || asc.samples != 1024) return SYMGPU_ERR_UNSUPPORTED;"),
        ("if (asc.object_type != 2 || asc.sbr_present || asc.channels > 2 || asc.samples != 1024) return SYMGPU_ERR_UNSUPPORTED;", "if (asc.object_type != 2 || asc.sbr_present || asc.channels > 2) return SYMGPU_ERR_UNSUPPORTED;"),
        ("case 35: case 36: case 37: case 38: case 39: case 40: case 41:", "case 35: case 36: case 37: case 38: case 39: case 40:"),
    ]),
    "vorbis": dict(src="vorbis_frontend.cpp", header="vorbis_entropy.h", prefix="symgpu_vorbis_fe_", tests=["tests/test_vorbis_frontend.py", "tests/test_zz_ogg_vorbis_to_pcm.py",
                                                                                     "tests/test_vorbis_codeword_fit.py"], mutants=[
        ("size_t k = (64 - left) >> 3;", "size_t k = (63 - left) >> 3;"),
        ("            needed -= left;\n            if (!fetch()) return false;", "            if (!fetch()) return false;\n            needed -= left > needed ? needed : left;"),
        ("if (left < 1 && !fetch()) return false;", "if (left < 2 && !fetch()) return false;"),
        ("if (bs.left < b.max_len) bs.top_up();", "if (bs.left <= b.max_len) bs.top_up();"),
        ("if (bs.left < b.max_len) bs.top_up();", "bs.top_up();"),
        ("if (depth + 1 > bs.left) return false;", "if (depth > bs.left) return false;"),
        ("if (free_nodes[k].depth > len) continue;", "if (free_nodes[k].depth >= len) continue;"),
        ("if (v < best_value) best_value = v, best = int(k);", "if (v <= best_value) best_value = v, best = int(k);"),
        ("return free_nodes.empty();", "return true;"),
        ("if (best < 0) return false;  // over-specified", "if (best < 0) continue;"),
        ("if (!bs.ok() || dims == 0 || dims > 32 || entries > 128 * 1024) return 1;", "if (!bs.ok() || dims == 0 || entries > 128 * 1024) return 1;"),
        ("if (lens.size() == 1 && lens[0] == 1)", "if (lens.size() == 1 && lens[0] == 2)"),
        ("if (!bs.ok() || lookup > 2) return 1;", "if (!bs.ok() || lookup > 3) return 1;"),
        ("if (sequence) last = v;", "if (!sequence) last = v;"),
        ("f.multiplier == 3 ? 86u", "f.multiplier == 3 ? 85u"),
        ("f.multiplier == 2 ? 128u", "f.multiplier == 2 ? 129u"),
        ("if (cbits && !read_code(S, S.books[cl.mainbook], bs, cval)) return false;", "if (!read_code(S, S.books[cl.mainbook], bs, cval)) return false;"),
        ("            cval >>= cbits;\n", ""),
        ("if (per_word > n_out) {", "if (per_word >= n_out) {"),
        ("element(rows, lanes, start + o) += v[k];", "element(rows, lanes, start + o) = v[k];"),
        ("for (size_t o = 0; o + dim <= n; o += dim) {", "for (size_t o = 0; o + dim < n; o += dim) {"),
        ("const size_t begin = min_sz(r.begin, full), end = min_sz(r.end, full);", "const size_t begin = r.begin, end = min_sz(r.end, full);"),
        ("const size_t begin = min_sz(r.begin, full), end = min_sz(r.end, full);", "const size_t begin = min_sz(r.begin, full), end = min_sz(r.end, n2);"),
        ("for (unsigned pass = 0; pass <= r.max_pass && !ended; ++pass)", "for (unsigned pass = 0; pass < r.max_pass && !ended; ++pass)"),
        ("                        if (r.type != 2 && do_not_decode[chans[c]]) continue;\n                        uint32_t code;", "                        uint32_t code;"),
        ("const size_t base = first + size_t(c) * parts;", "const size_t base = first;"),
        ("cls.size - base);", "parts - first);"),
        ("if (!(r.used[k] & (1u << pass))) continue;", "if (!(r.used[k] & (1u << pass)) && pass) continue;"),
        ("rows[j & 1][j >> 1]", "rows[(j >> 1) & 1][j >> 1]"),
        ("if (fe) fe->prev_block_flag = -1;", ""),
        ("if (!bs.read_bool(flag) || flag) return SYMGPU_ERR_DECODE;  // lib.rs:151-154", "if (!bs.read_bool(flag)) return SYMGPU_ERR_DECODE;"),
        ("|| mode_number >= n_modes) return SYMGPU_ERR_DECODE;", ") return SYMGPU_ERR_DECODE;"),
        ("if (!bs.read_bool(flag) || !bs.read_bool(flag)) return SYMGPU_ERR_DECODE;", "if (!bs.read_bool(flag)) return SYMGPU_ERR_DECODE;"),
        ("if (mapping.coupled && unit->do_not_decode[0] != unit->do_not_decode[1]) unit->do_not_decode[0] = unit->do_not_decode[1] = 0;", ""),
        ("        if (!used)\n            for (int i = 0; i < 65; ++i) floor_y[ch * 65 + i] = 0;\n", ""),
    ]),
}

DRIVER = r'''
import ctypes, sys
sys.path.insert(0, {root!r})
from symphonia_b200 import _native as nat
real = nat.lib()
mut = ctypes.CDLL({so!r})
class Proxy:
    def __getattr__(self, name):
        if name.startswith({prefix!r}):
            f, g = getattr(mut, name), getattr(real, name)
            f.argtypes, f.restype = g.argtypes, g.restype
            return f
        return getattr(real, name)
proxy = Proxy()
nat.lib = lambda: proxy
import pytest
sys.exit(pytest.main(["-x", "-q", "-p", "no:cacheprovider", "-m", "not gpu"] + {tests!r}))
'''


def main():
    t = TARGETS[sys.argv[1]]
    src = open(os.path.join(CSRC, t["src"])).read()
    # rules shared with a device decoder live in a header the source includes: a mutant found there is applied to a copy of
    # the header, and the source's copy includes that copy instead
    header = open(os.path.join(CSRC, t["header"])).read() if "header" in t else ""
    survivors = []
    with tempfile.TemporaryDirectory() as tmp:
        for k, (old, new) in enumerate(t["mutants"]):
            in_src = src.count(old) >= 1
            assert in_src or header.count(old) >= 1, old
            path = os.path.join(CSRC, f"_mutant_{k}.cpp")  # next to the original: relative includes
            hpath = os.path.join(CSRC, f"_mutant_{k}.h")
            so = os.path.join(tmp, f"m{k}.so")
            with open(path, "w") as f:
                f.write(src.replace(old, new, 1) if in_src else src.replace(f'#include "{t["header"]}"', f'#include "_mutant_{k}.h"'))
            if not in_src:
                with open(hpath, "w") as f:
                    f.write(header.replace(old, new, 1))
            try:
                cc = subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-I/usr/local/cuda/include", "-o", so, path] +
                                    ([os.path.join(CSRC, "packetizer.cpp")] if sys.argv[1] == "vorbis" else []), capture_output=True, text=True)
            finally:
                os.remove(path)
                if os.path.exists(hpath):
                    os.remove(hpath)
            if cc.returncode:
                print(f"[{k}] does not compile: {old!r}")
                continue
            drv = os.path.join(tmp, "drv.py")
            with open(drv, "w") as f:
                f.write(DRIVER.format(root=ROOT, so=so, prefix=t["prefix"], tests=[os.path.join(ROOT, x) for x in t["tests"]]))
            try:
                res = subprocess.run([sys.executable, drv], capture_output=True, text=True, timeout=600, cwd=ROOT)
                killed = res.returncode != 0
            except subprocess.TimeoutExpired:
                killed = True
            print(f"[{k}] {'killed  ' if killed else 'SURVIVED'} {old!r} -> {new!r}", flush=True)
            if not killed:
                survivors.append((old, new))
    print(f"{len(t['mutants']) - len(survivors)} of {len(t['mutants'])} killed; survivors: {len(survivors)}")


if __name__ == "__main__":
    main()
