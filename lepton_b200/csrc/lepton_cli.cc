// lepton_cli.cc -- `lepton`-compatible command line front end over liblepton_b200.so.
//
// Keeps the part of the reference CLI surface that selects what is computed (src/lepton/jpgcoder.cc
// initialize_options :988-1219, process_file :1528): `lepton [flags] <in.jpg|in.lep> [out]`, direction chosen from
// the first two bytes of the input (FF D8 -> compress, CF 84 or CE B6 -> decompress; check_file :2178), `-` for stdin/stdout,
// exit status = the reference's ExitCode (src/vp8/util/memory.hh:13-39).  Flags that only configure the reference's
// CPU runtime (-singlethread, -unjailed, -preload, -memory=, -threadmemory=, -timebound=) are accepted and ignored.
// Like the reference, the CLI verifies every .lep it writes by decoding it again (exit code 41, ROUNDTRIP_FAILURE, and no
// output when the input does not come back byte for byte) unless -skipverify is given.  Service modes (-socket, -listen, -fork,
// -benchmark, -lepcat) and output variants this build does not write (-brotliheader, -ans, -ujg, -startbyte / -trunc slices)
// are refused, never silently ignored.  Flags that change the bytes are honoured:
// -minencodethreads= / -maxencodethreads= / -evensplit (thread-segment selection), -rejectprogressive / -allowprogressive,
// -zlib0: a restored JPEG is written as a zlib stream of stored blocks (jpgcoder.cc:2089, 2200-2220), default name
// <stem>.jpg.z (open_fdout, jpgcoder.cc:1477-1479).  A .lep whose magic is CE B6 (zeta) is always restored that way; the
// JPEG -> .lep direction ignores -zlib0.
// -embedding=N: every input is a JPEG whose SOI sits at byte N of the file, whatever its first two bytes (check_file,
// jpgcoder.cc:2192); the N bytes in front of it are kept in the .lep and come back in front of the JPEG on restore.
// -d: the .lep keeps only the header segments the coefficients are coded with (rebuild_header_jpg, jpgcoder.cc:4848).
// -permissive: every input is compressed, whatever its first bytes and however short (jpgcoder.cc:1472, 1603), and verified
// even with -skipverify; a file the coder cannot take -- or whose .lep would not restore it -- is stored whole in the
// reference's generic container ('Y'), which restores it byte for byte.  Only an empty input still fails (42).
// A .lep input may be a stream of concatenated .lep files (`cat a.lep b.lep | lepton-b200 -`, the reference's -lepcat files;
// process_file, jpgcoder.cc:1867-1898): it is restored to the members' JPEGs one after the other, in single-file, stdin and
// batch mode alike.  Writing -lepcat and -brotliheader files stays refused: both need brotli output identical to the
// reference's vendored brotli 1.0.0, and the system's libbrotlienc 1.1.0 with the reference's BrotliCodec::Compress settings
// gave other bytes in 40 of 81 compressions of this repository's files at quality 9-11.
//
// Batch mode (no reference counterpart; a GPU wants thousands of files per call, the reference one per process):
//   lepton-b200 -outdir=DIR [-devices=0,1,...] a.jpg b.lep c.jpg ...
// every positional argument is an input, the direction is chosen per file, all JPEGs go through ONE
// lepb200_compress_jpegs call and all .lep files through ONE lepb200_decompress_leps call; outputs are DIR/<name>.lep /
// DIR/<name>.jpg (DIR/<name>.jpg.z for zlib0 output).  With -devices= the files are dealt to one codec per GPU, balanced by bytes (lepb200_*_multi).  A file that fails reports its ExitCode on stderr and does not stop the others; the exit status is
// the first non-zero one.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <string>
#include <thread>
#include <vector>

#include "../../include/lepton_b200.h"

static bool read_all(FILE* f, std::vector<uint8_t>& out) {
    uint8_t buf[1 << 16];
    size_t n;
    while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out.insert(out.end(), buf, buf + n);
    return !ferror(f);
}

static std::string base_name(const std::string& path) {
    size_t slash = path.find_last_of('/');
    std::string b = slash == std::string::npos ? path : path.substr(slash + 1);
    size_t dot = b.rfind('.');
    if (dot != std::string::npos && dot > 0) b.resize(dot);
    return b;
}

// -outdir=DIR: all inputs in two library calls (one per direction)
static bool is_lep_magic(const std::vector<uint8_t>& d) { return (d[0] == 0xCF && d[1] == 0x84) || (d[0] == 0xCE && d[1] == 0xB6); }

static int run_batch(const std::vector<std::string>& files, const std::string& outdir, const std::vector<int>& devices, int allow_progressive, int min_threads, int max_threads, int even_split, int verify, int zlib0,
                     long long embedding, int discard_meta, int permissive) {
    struct Item { std::string name; std::vector<uint8_t> data; bool is_jpeg = false, zeta = false; int status = 0; };
    std::vector<Item> items(files.size());
    int first_err = 0;
    for (size_t i = 0; i < files.size(); ++i) {
        Item& it = items[i];
        it.name = files[i];
        FILE* f = fopen(files[i].c_str(), "rb");
        if (!f) { it.status = 9; }                                                               // FILE_NOT_FOUND
        else {
            if (!read_all(f, it.data)) it.status = 33;
            fclose(f);
            if (!it.status && it.data.size() < 2 && !permissive) it.status = 3;                      // SHORT_READ
        }
        if (!it.status) {
            it.is_jpeg = permissive || embedding >= 0 || (it.data[0] == 0xFF && it.data[1] == 0xD8);
            it.zeta = !it.is_jpeg && it.data[0] == 0xCE && it.data[1] == 0xB6;
            if (!it.is_jpeg && !is_lep_magic(it.data)) it.status = 42;                              // UNSUPPORTED_JPEG
        }
    }
    // one codec per GPU; the host threads are divided between them
    std::vector<lepb200_codec*> codecs;
    auto destroy_all = [&]() { for (lepb200_codec* c : codecs) lepb200_codec_destroy(c); };
    const int host_threads = devices.size() > 1 ? (int)std::max<size_t>(1, std::thread::hardware_concurrency() / devices.size()) : 0;
    int rc = 0;
    for (int dev : devices) {
        lepb200_codec* c = nullptr;
        rc = lepb200_codec_create(&c, dev, host_threads);
        if (rc) { fprintf(stderr, "lepton-b200: no usable CUDA device %d (%d); this build has no CPU coder\n", dev, rc); destroy_all(); return 33; }
        lepb200_codec_set_allow_progressive(c, allow_progressive);
        lepb200_codec_set_encode_threads(c, min_threads, max_threads);
        lepb200_codec_set_even_split(c, even_split);
        lepb200_codec_set_verify(c, verify);
        lepb200_codec_set_zlib0(c, zlib0);
        lepb200_codec_set_embedding(c, embedding);
        lepb200_codec_set_discard_meta(c, discard_meta);
        lepb200_codec_set_permissive(c, permissive);
        codecs.push_back(c);
    }
    for (int dir = 0; dir < 2; ++dir) {                      // 0: JPEG -> .lep, 1: .lep -> JPEG
        std::vector<size_t> idx;
        std::vector<lepb200_buffer> in;
        for (size_t i = 0; i < items.size(); ++i)
            if (!items[i].status && items[i].is_jpeg == (dir == 0)) { idx.push_back(i); in.push_back({items[i].data.data(), items[i].data.size()}); }
        if (idx.empty()) continue;
        std::vector<lepb200_result> res(idx.size(), lepb200_result{nullptr, 0, 0});
        rc = dir == 0 ? lepb200_compress_jpegs_multi(codecs.data(), (int)codecs.size(), in.data(), (int)in.size(), res.data())
                      : lepb200_decompress_leps_multi(codecs.data(), (int)codecs.size(), in.data(), (int)in.size(), res.data());
        if (rc) {
            for (lepb200_codec* c : codecs) { const char* e = lepb200_codec_last_error(c); if (e && *e) fprintf(stderr, "lepton-b200: %s\n", e); }
            destroy_all();
            return 33;
        }
        for (size_t k = 0; k < idx.size(); ++k) {            // results stay valid until the next call on the codec: write now
            Item& it = items[idx[k]];
            it.status = res[k].status == LEPB200_ST_NOT_HANDLED ? 42 : res[k].status;
            if (it.status) continue;
            const std::string out = outdir + "/" + base_name(it.name) + (dir == 0 ? ".lep" : (zlib0 || it.zeta) ? ".jpg.z" : ".jpg");
            FILE* fo = fopen(out.c_str(), "wb");
            if (!fo || fwrite(res[k].data, 1, res[k].len, fo) != res[k].len) it.status = 33;
            if (fo) fclose(fo);
        }
    }
    destroy_all();
    for (const Item& it : items) {
        if (!it.status) continue;
        fprintf(stderr, "lepton-b200: %s: exit code %d\n", it.name.c_str(), it.status);
        if (!first_err) first_err = it.status;
    }
    return first_err;
}

int main(int argc, char** argv) {
    std::vector<std::string> files;
    std::string outdir;
    int device = 0;
    std::vector<int> devices;
    int even_split = 0;
    int verify = 1;              // the reference verifies every file it writes unless told -skipverify (jpgcoder.cc:107-112, 1095-1110)
    int min_threads = 1, max_threads = 8;   // -minencodethreads= / -maxencodethreads=: bounds of the thread-segment count (change the .lep bytes)
    int allow_progressive = 1;   // this build follows the reference compiled with DEFAULT_ALLOW_PROGRESSIVE (CMakeLists.txt:293)
    int zlib0 = 0;               // -zlib0: restored JPEGs are written as zlib streams
    long long embedding = -1;    // -embedding=N: inputs are JPEGs at byte N of a larger file
    int discard_meta = 0;        // -d: metadata segments are left out of the .lep
    int permissive = 0;          // -permissive: files the coder cannot take go into the generic container
    for (int i = 1; i < argc; ++i) {
        const char* a = argv[i];
        if (a[0] == '-' && a[1] != 0) {
            if (!strncmp(a, "-device=", 8)) { device = atoi(a + 8); continue; }
            if (!strncmp(a, "-devices=", 9)) {                       // batch mode on several GPUs: -devices=0,1,2,3
                for (const char* q = a + 9; *q;) { devices.push_back(atoi(q)); while (*q && *q != ',') ++q; if (*q == ',') ++q; }
                continue;
            }
            if (!strncmp(a, "-outdir=", 8)) { outdir = a + 8; continue; }
            if (!strncmp(a, "-minencodethreads=", 18)) { min_threads = atoi(a + 18); continue; }
            if (!strncmp(a, "-maxencodethreads=", 18)) { max_threads = atoi(a + 18); continue; }
            if (!strcmp(a, "-evensplit")) { even_split = 1; continue; }
            if (!strcmp(a, "-skipverify") || !strcmp(a, "-skipverification") || !strcmp(a, "-skiproundtrip")) { verify = 0; continue; }
            if (!strcmp(a, "-verify") || !strcmp(a, "-verification") || !strcmp(a, "-roundtrip") || !strcmp(a, "-validate") ||
                !strcmp(a, "-validation")) { verify = 1; continue; }
            if (!strcmp(a, "-rejectprogressive")) { allow_progressive = 0; continue; }
            if (!strcmp(a, "-zlib0")) { zlib0 = 1; continue; }
            if (!strncmp(a, "-embedding=", 11)) { embedding = std::max(0ll, atoll(a + 11)); continue; }
            if (!strcmp(a, "-d")) { discard_meta = 1; continue; }
            if (!strcmp(a, "-permissive")) { permissive = 1; continue; }
            if (!strcmp(a, "-allowprogressive") || !strcmp(a, "-forceprogressive")) { allow_progressive = 1; continue; }
            if (!strcmp(a, "-socket") || !strncmp(a, "-socket=", 8) || !strncmp(a, "-listen", 7) || !strcmp(a, "-fork") ||
                !strcmp(a, "-benchmark") || !strcmp(a, "-lepcat") || !strncmp(a, "-startbyte", 10) || !strncmp(a, "-trunc=", 7) ||
                !strcmp(a, "-ujg") || !strcmp(a, "-brotliheader") || !strcmp(a, "-ans")) {
                fprintf(stderr, "lepton-b200: option %s is outside this build\n", a);
                return 13;   // VERSION_UNSUPPORTED
            }
            continue;        // runtime-tuning flags of the CPU reference: accepted, no effect
        }
        files.push_back(a);
    }
    if (files.empty()) {
        fprintf(stderr, "usage: lepton-b200 [flags] <input.jpg|input.lep|-> [output|-]\n"
                        "       lepton-b200 [flags] -outdir=DIR <inputs...>      (one batch per direction)\n");
        return 1;
    }
    if (devices.empty()) devices.push_back(device);
    if (!outdir.empty()) return run_batch(files, outdir, devices, allow_progressive, min_threads, max_threads, even_split, verify, zlib0, embedding, discard_meta, permissive);
    std::vector<uint8_t> in;
    FILE* fi = files[0] == "-" ? stdin : fopen(files[0].c_str(), "rb");
    if (!fi) { fprintf(stderr, "lepton-b200: cannot open %s\n", files[0].c_str()); return 9; }   // FILE_NOT_FOUND
    if (!read_all(fi, in)) return 33;                                                            // OS_ERROR
    if (fi != stdin) fclose(fi);
    if (in.size() < 2 && !permissive) return 3;                                                  // SHORT_READ
    const bool is_jpeg = permissive || embedding >= 0 || (in[0] == 0xFF && in[1] == 0xD8), is_lep = !is_jpeg && is_lep_magic(in);
    const bool zlib_out = is_lep && (zlib0 || (in[0] == 0xCE && in[1] == 0xB6));
    if (!is_jpeg && !is_lep) { fprintf(stderr, "lepton-b200: input is neither JPEG nor Lepton\n"); return 42; }
    std::string outname;
    if (files.size() > 1) outname = files[1];
    else if (files[0] == "-") outname = "-";
    else {
        outname = files[0];
        size_t dot = outname.rfind('.');
        if (dot != std::string::npos) outname.resize(dot);
        outname += is_jpeg ? ".lep" : zlib_out ? ".jpg.z" : ".jpg";
    }
    lepb200_codec* codec = nullptr;
    int rc = lepb200_codec_create(&codec, device, 0);
    if (rc) { fprintf(stderr, "lepton-b200: no usable CUDA device (%d); this build has no CPU coder\n", rc); return 33; }
    lepb200_codec_set_allow_progressive(codec, allow_progressive);
    lepb200_codec_set_encode_threads(codec, min_threads, max_threads);
    lepb200_codec_set_even_split(codec, even_split);
    lepb200_codec_set_verify(codec, verify);
    lepb200_codec_set_zlib0(codec, zlib0);
    lepb200_codec_set_embedding(codec, embedding);
    lepb200_codec_set_discard_meta(codec, discard_meta);
    lepb200_codec_set_permissive(codec, permissive);
    lepb200_buffer ib = {in.data(), in.size()};
    lepb200_result res = {nullptr, 0, 0};
    rc = is_jpeg ? lepb200_compress_jpegs(codec, &ib, 1, &res) : lepb200_decompress_leps(codec, &ib, 1, &res);
    if (rc) { fprintf(stderr, "lepton-b200: %s\n", lepb200_codec_last_error(codec)); lepb200_codec_destroy(codec); return 33; }
    if (res.status) {
        fprintf(stderr, "lepton-b200: exit code %d\n", res.status);
        lepb200_codec_destroy(codec);
        return res.status == LEPB200_ST_NOT_HANDLED ? 42 : res.status;
    }
    FILE* fo = outname == "-" ? stdout : fopen(outname.c_str(), "wb");
    if (!fo) { lepb200_codec_destroy(codec); return 33; }
    bool wrote = fwrite(res.data, 1, res.len, fo) == res.len;
    if (fo != stdout) wrote = (fclose(fo) == 0) && wrote; else wrote = (fflush(fo) == 0) && wrote;
    if (!wrote) { fprintf(stderr, "lepton-b200: could not write %s\n", outname.c_str()); lepb200_codec_destroy(codec); return 33; }     // OS_ERROR
    if (is_jpeg) fprintf(stderr, "%zu %zu\n%.2f%%\n", res.len, in.size(), 100.0 * (double)res.len / (double)in.size());
    lepb200_codec_destroy(codec);
    return 0;
}
