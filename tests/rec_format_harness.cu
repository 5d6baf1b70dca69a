// Host harness for rechorus_b200/csrc/rec_format.cuh: formats every value of a binary file, one text per line.
//
//     rec_format_harness f32|i64 <style> <in.bin> <out.txt>
//
// f32 reads little-endian uint32 float bit patterns, i64 reads int64 values; style is B2R_REC_STYLE_NP (0) or
// B2R_REC_STYLE_BARE (1).  tests/test_rec_csv_cpu.py compiles it with nvcc and compares the lines with NumPy's repr.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../rechorus_b200/csrc/rec_format.cuh"

int main(int argc, char** argv) {
    if (argc != 5 || (strcmp(argv[1], "f32") && strcmp(argv[1], "i64"))) {
        fprintf(stderr, "usage: %s f32|i64 style in.bin out.txt\n", argv[0]);
        return 2;
    }
    const bool f32 = strcmp(argv[1], "f32") == 0;
    const int style = atoi(argv[2]);
    FILE* in = fopen(argv[3], "rb");
    FILE* out = fopen(argv[4], "wb");
    if (!in || !out) {
        fprintf(stderr, "cannot open %s or %s\n", argv[3], argv[4]);
        return 1;
    }
    static char buf[1 << 16];
    size_t fill = 0;
    char text[b2r::recfmt::kMaxText + 1];
    for (;;) {
        int n;
        if (f32) {
            uint32_t bits;
            if (fread(&bits, sizeof bits, 1, in) != 1) break;
            n = b2r::recfmt::format_f32(bits, style, text);
        } else {
            int64_t v;
            if (fread(&v, sizeof v, 1, in) != 1) break;
            n = b2r::recfmt::format_i64(v, style, text);
        }
        if (fill + n + 1 > sizeof buf) {
            fwrite(buf, 1, fill, out);
            fill = 0;
        }
        memcpy(buf + fill, text, n);
        fill += n;
        buf[fill++] = '\n';
    }
    fwrite(buf, 1, fill, out);
    fclose(in);
    return fclose(out) == 0 ? 0 : 1;
}
