// Both DEFLATE decoders of the project -- the host's (csrc/host/inflate_fast.hpp) and the bit-stream half of the device's
// (csrc/vtx_inflate.cuh, through tests/inflate_dev_shim.cpp) -- over a file of crafted streams, built with
// -fsanitize=address,undefined by tests/test_deflate_craft_cpu.py.  A decoder that reads or writes outside its buffers on
// any stream, valid or not, stops the run here instead of faulting on the device.
//   usage: inflate_asan CORPUS
//   CORPUS: records of  u32 in_len, u32 out_len, u32 valid, in_len bytes of stream, (valid ? out_len bytes of output : nothing)
#include <cstdio>
#include <cstring>
#include <vector>

#include "inflate_dev_shim.cpp"
#include "inflate_shim.cpp"

int main(int argc, char** argv)
{
    if (argc < 2) { fprintf(stderr, "usage: %s CORPUS\n", argv[0]); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<unsigned char> d;
    unsigned char buf[1 << 16];
    size_t n;
    while ((n = fread(buf, 1, sizeof(buf), f)) > 0) d.insert(d.end(), buf, buf + n);
    fclose(f);
    size_t p = 0;
    long n_ok = 0, n_refused = 0, bad = 0;
    while (p + 12 <= d.size()) {
        uint32_t in_len, out_len, valid;
        memcpy(&in_len, &d[p], 4); memcpy(&out_len, &d[p + 4], 4); memcpy(&valid, &d[p + 8], 4); p += 12;
        // exactly-sized heap copies: the sanitizer sees any read past the stream's promised padding
        std::vector<unsigned char> in(d.begin() + long(p), d.begin() + long(p + in_len));
        p += in_len;
        in.resize(in_len + vtxhost::kInflateInPad, 0xAA);
        std::vector<unsigned char> host_out(out_len + vtxhost::kInflateOutPad), dev_out(out_len + 8);
        const bool host_ok = vtx_test_inflate(in.data(), in_len, host_out.data(), out_len) != 0;
        std::vector<unsigned char> in_exact(in.begin(), in.begin() + in_len);
        const int dev_st = vtx_test_inflate_dev(in_exact.data(), in_len, dev_out.data(), out_len);
        if (valid) {
            const unsigned char* want = &d[p];
            p += out_len;
            if (!host_ok || memcmp(host_out.data(), want, out_len) != 0) { printf("host decoder differs from zlib at record %ld\n", n_ok + n_refused); ++bad; }
            if (dev_st != 0 || memcmp(dev_out.data(), want, out_len) != 0) { printf("device logic differs from zlib at record %ld (status %d)\n", n_ok + n_refused, dev_st); ++bad; }
            ++n_ok;
        } else {
            if (host_ok) { printf("host decoder accepts invalid record %ld\n", n_ok + n_refused); ++bad; }
            if (dev_st == 0) { printf("device logic accepts invalid record %ld\n", n_ok + n_refused); ++bad; }
            ++n_refused;
        }
    }
    printf("valid %ld, invalid %ld, disagreements %ld\n", n_ok, n_refused, bad);
    return bad ? 1 : 0;
}
