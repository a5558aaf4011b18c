// ref_harness_interleaved.cpp -- the REFERENCE's own FastqReaderPair over an interleaved file (TEST INFRASTRUCTURE,
// oracle/_ref/libfastp_ref_interleaved.so, built by __graft_entry__.build() against the reference objects in oracle/_ref/libfastp_ref.so).
// Used to pin the C port of interleaved reading (oracle/fastp_oracle_interleaved.c) in tests/test_oracle_fastq_interleaved.py.
#include <cstdint>
#include <cstring>
#include <string>
#include "read.h"
#include "fastqreader.h"

extern "C" {

// FastqReaderPair(path, "", true, phred64, interleaved = true) (src/fastqreader.cpp:432-460): every pair it returns until ReadPair::eof
// (src/read.cpp:203-205), each pair as two records flattened as [name_len, seq_len, strand_len, qual_len] (4 x int32) followed by the four
// byte strings.  Returns the pair count; *used = bytes written (nothing is written past cap, the count still runs on).
int64_t fp_ref_fastq_read_interleaved(const char* path, int phred64, uint8_t* out, int64_t cap, int64_t* used) {
    FastqReaderPair reader(path, "", true, phred64 != 0, true);
    int64_t n = 0, o = 0;
    for (;;) {
        ReadPair* p = new ReadPair();
        reader.read(p);
        if (p->eof()) { delete p; break; }
        for (Read* r : {p->mLeft, p->mRight}) {
            const std::string* f[4] = {r->mName, r->mSeq, r->mStrand, r->mQuality};
            int64_t need = 16;
            for (int k = 0; k < 4; k++) need += (int64_t)f[k]->size();
            if (o + need <= cap) {
                int32_t* h = reinterpret_cast<int32_t*>(out + o);
                for (int k = 0; k < 4; k++) h[k] = (int32_t)f[k]->size();
                uint8_t* d = out + o + 16;
                for (int k = 0; k < 4; k++) { memcpy(d, f[k]->data(), f[k]->size()); d += f[k]->size(); }
            }
            o += need;
        }
        n++;
        delete p;
    }
    *used = o;
    return n;
}

}  // extern "C"
