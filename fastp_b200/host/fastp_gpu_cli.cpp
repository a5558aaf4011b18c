/*
 * fastp_gpu_cli.cpp -- minimal plain-FASTQ driver around GpuChainWorker (the caller either side of the hot path,
 * SURVEY.md 8(f) rank 1 kept on the host for now): reads R1[/R2], packs reads like the reference's reader
 * (src/peprocessor.cpp:760-813), runs the device chain through the drop-in bodies, writes the passing reads and a
 * small JSON summary.  Flags are the reference's own spellings (src/main.cpp:32-158) for the options the chain reads.
 */
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <string>
#include <sys/stat.h>
#include <vector>
#include "fastp_host.h"

using namespace fastp_b200;

/* Options::makeListFromFileByLine (src/options.cpp:484-510) after check_file_valid (src/util.h:185-194): one barcode per line read with
   getline(line, 1000) -- a line of 1000 bytes or more ends the list there --, a trailing '\r' (or "\r\r") dropped only from lines of two
   bytes or more, and any byte other than A/T/C/G ends the run.  Exit status and messages are the reference's. */
static std::vector<std::string> loadBarcodes(const std::string& filename) {
    struct stat st;
    if (stat(filename.c_str(), &st) != 0) { std::cerr << "ERROR: file '" << filename << "' doesn't exist, quit now" << std::endl; exit(-1); }
    if (S_ISDIR(st.st_mode)) { std::cerr << "ERROR: '" << filename << "' is a folder, not a file, quit now" << std::endl; exit(-1); }
    std::vector<std::string> ret;
    std::ifstream file(filename.c_str(), std::ifstream::in);
    const int maxLine = 1000;
    char line[maxLine];
    std::cerr << "filter by index, loading " << filename << std::endl;
    while (file.getline(line, maxLine)) {
        const size_t got = strlen(line);             /* the line up to its first NUL byte, as the reference sees it */
        if (got >= 2 && (line[got - 1] == '\n' || line[got - 1] == '\r')) {
            line[got - 1] = '\0';
            if (line[got - 2] == '\r') line[got - 2] = '\0';
        }
        const std::string bc(line);
        for (char ch : bc)
            if (ch != 'A' && ch != 'T' && ch != 'C' && ch != 'G') {
                std::cerr << "ERROR: processing " << filename << ", each line should be one barcode, which can only contain A/T/C/G" << std::endl;
                exit(-1);
            }
        std::cerr << bc << std::endl;
        ret.push_back(bc);
    }
    std::cerr << std::endl;
    return ret;
}

static Read* readRecord(std::istream& in) {          /* FastqReader::read src/fastqreader.cpp:309-368 (plain text only) */
    std::string name, seq, strand, qual;
    if (!std::getline(in, name)) return nullptr;
    while (name.empty()) if (!std::getline(in, name)) return nullptr;
    if (!std::getline(in, seq) || !std::getline(in, strand) || !std::getline(in, qual)) return nullptr;
    if (name[0] != '@' || seq.size() != qual.size()) return nullptr;
    return new Read(new std::string(name), new std::string(seq), new std::string(strand), new std::string(qual));
}

int main(int argc, char** argv) {
    Options opt;
    std::string in1, in2, out1, out2, mergedOut, unpaired1, unpaired2, failedOut, overlappedOut, json, indexList1, indexList2;
    int packSize = 1 << 16, maxLen = 0;
    bool deviceFastq = false, phred64 = false;
    bool interleavedIn = false, fromStdin = false, toStdout = false;     /* src/main.cpp:194-196 */
    bool dedup = false, evalDup = true; int dupLevel = 0;     /* src/main.cpp:200-209 */
    int zlevel = 4, zthreads = 8;          /* -z / --compression (src/main.cpp:50), host threads for .gz output */
    size_t chunkBytes = 0;                 /* text path: bytes read per side per step (default: about one device batch) */
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        auto next = [&]() -> const char* { if (i + 1 >= argc) { fprintf(stderr, "missing value for %s\n", a.c_str()); exit(2); } return argv[++i]; };
        if (a == "-i" || a == "--in1") in1 = next(); else if (a == "-I" || a == "--in2") in2 = next();
        else if (a == "-o" || a == "--out1") out1 = next(); else if (a == "-O" || a == "--out2") out2 = next();
        else if (a == "--unpaired1") unpaired1 = next(); else if (a == "--unpaired2") unpaired2 = next();
        else if (a == "--failed_out") failedOut = next();
        else if (a == "--overlapped_out") overlappedOut = next();
        else if (a == "--filter_by_index1") indexList1 = next(); else if (a == "--filter_by_index2") indexList2 = next();
        else if (a == "--filter_by_index_threshold") opt.indexFilter.threshold = atoi(next());
        else if (a == "-j" || a == "--json") json = next();
        else if (a == "-A" || a == "--disable_adapter_trimming") opt.adapter.enabled = false;
        else if (a == "-a" || a == "--adapter_sequence") { opt.adapter.sequence = next(); opt.adapter.hasSeqR1 = true; }
        else if (a == "--adapter_sequence_r2") { opt.adapter.sequenceR2 = next(); opt.adapter.hasSeqR2 = true; }
        else if (a == "-f" || a == "--trim_front1") opt.trim.front1 = atoi(next()); else if (a == "-t" || a == "--trim_tail1") opt.trim.tail1 = atoi(next());
        else if (a == "-F" || a == "--trim_front2") opt.trim.front2 = atoi(next()); else if (a == "-T" || a == "--trim_tail2") opt.trim.tail2 = atoi(next());
        else if (a == "-b" || a == "--max_len1") opt.trim.maxLen1 = atoi(next()); else if (a == "-B" || a == "--max_len2") opt.trim.maxLen2 = atoi(next());
        else if (a == "-g" || a == "--trim_poly_g") opt.polyGTrim.enabled = true; else if (a == "--poly_g_min_len") opt.polyGTrim.minLen = atoi(next());
        else if (a == "-x" || a == "--trim_poly_x") opt.polyXTrim.enabled = true; else if (a == "--poly_x_min_len") opt.polyXTrim.minLen = atoi(next());
        else if (a == "-5" || a == "--cut_front") opt.qualityCut.enabledFront = true; else if (a == "-3" || a == "--cut_tail") opt.qualityCut.enabledTail = true;
        else if (a == "-r" || a == "--cut_right") opt.qualityCut.enabledRight = true;
        else if (a == "-W" || a == "--cut_window_size") { int w = atoi(next()); opt.qualityCut.windowSizeFront = opt.qualityCut.windowSizeTail = opt.qualityCut.windowSizeRight = w; }
        else if (a == "-M" || a == "--cut_mean_quality") { int q = atoi(next()); opt.qualityCut.qualityFront = opt.qualityCut.qualityTail = opt.qualityCut.qualityRight = q; }
        else if (a == "-Q" || a == "--disable_quality_filtering") opt.qualfilter.enabled = false;
        else if (a == "-q" || a == "--qualified_quality_phred") opt.qualfilter.qualifiedQual = (char)(33 + atoi(next()));
        else if (a == "-u" || a == "--unqualified_percent_limit") opt.qualfilter.unqualifiedPercentLimit = atoi(next());
        else if (a == "-n" || a == "--n_base_limit") opt.qualfilter.nBaseLimit = atoi(next()); else if (a == "-e" || a == "--average_qual") opt.qualfilter.avgQualReq = atoi(next());
        else if (a == "-L" || a == "--disable_length_filtering") opt.lengthFilter.enabled = false;
        else if (a == "-l" || a == "--length_required") opt.lengthFilter.requiredLength = atoi(next()); else if (a == "--length_limit") opt.lengthFilter.maxLength = atoi(next());
        else if (a == "-y" || a == "--low_complexity_filter") opt.complexityFilter.enabled = true;
        else if (a == "-Y" || a == "--complexity_threshold") opt.complexityFilter.threshold = std::min(100, std::max(0, atoi(next()))) / 100.0;
        else if (a == "-c" || a == "--correction") opt.correction.enabled = true;
        else if (a == "-m" || a == "--merge") opt.merge.enabled = true; else if (a == "--merged_out") mergedOut = next();
        else if (a == "--include_unmerged") opt.merge.includeUnmerged = true;
        else if (a == "--overlap_len_require") opt.overlapRequire = atoi(next()); else if (a == "--overlap_diff_limit") opt.overlapDiffLimit = atoi(next());
        else if (a == "--overlap_diff_percent_limit") opt.overlapDiffPercentLimit = atoi(next());
        else if (a == "--interleaved_in") interleavedIn = true; else if (a == "--stdin") fromStdin = true; else if (a == "--stdout") toStdout = true;
        else if (a == "--device_fastq") deviceFastq = true; else if (a == "-6" || a == "--phred64") phred64 = true;
        else if (a == "--chunk_bytes") chunkBytes = (size_t)atoll(next());
        else if (a == "-D" || a == "--dedup") dedup = true; else if (a == "--dup_calc_accuracy") dupLevel = std::min(6, std::max(1, atoi(next())));
        else if (a == "--dont_eval_duplication") evalDup = false;
        else if (a == "-z" || a == "--compression") zlevel = std::min(9, std::max(1, atoi(next()))); else if (a == "--zthreads") zthreads = std::max(1, atoi(next()));
        else if (a == "--max_read_len") maxLen = atoi(next()); else if (a == "--pack_size") packSize = atoi(next());
        else { fprintf(stderr, "unknown flag %s\n", a.c_str()); return 2; }
    }
    if (in1.empty() && fromStdin && in2.empty()) in1 = "/dev/stdin";    /* src/options.cpp:85-93 */
    if (in1.empty()) { fprintf(stderr, "usage: fastp_gpu_cli -i R1.fq [-I R2.fq] [--interleaved_in] [--stdin] [--stdout] [-o out1.fq] [-O out2.fq] [-m --merged_out merged.fq] [--unpaired1 u1.fq] [--unpaired2 u2.fq] [--failed_out failed.fq] [--overlapped_out ov.fq] [--filter_by_index1 list] [--filter_by_index2 list] [-j summary.json] [fastp flags]\n"); return 2; }
    if (!deviceFastq && (interleavedIn || fromStdin || toStdout)) { fprintf(stderr, "ERROR: --interleaved_in / --stdin / --stdout need --device_fastq\n"); return 2; }
    const bool stdinInput = in1 == "/dev/stdin";         /* read as it comes: nothing may open it twice */
    if (toStdout) {                                      /* src/options.cpp:101-110 */
        if (!out1.empty()) { std::cerr << "In STDOUT mode, ignore the out1 filename " << out1 << std::endl; out1.clear(); }
        if (!out2.empty()) { std::cerr << "In STDOUT mode, ignore the out2 filename " << out2 << std::endl; out2.clear(); }
    }
    opt.paired = !in2.empty() || interleavedIn;
    if (!deviceFastq && !(unpaired1.empty() && unpaired2.empty() && failedOut.empty())) {
        fprintf(stderr, "ERROR: --unpaired1 / --unpaired2 / --failed_out need --device_fastq\n"); return 2;
    }
    if (!deviceFastq && !overlappedOut.empty()) { fprintf(stderr, "ERROR: --overlapped_out needs --device_fastq\n"); return 2; }
    if (!deviceFastq && !(indexList1.empty() && indexList2.empty())) { fprintf(stderr, "ERROR: --filter_by_index1 / --filter_by_index2 need --device_fastq\n"); return 2; }
    if (unpaired2.empty()) unpaired2 = unpaired1;       /* src/main.cpp:188-189 */
    auto fail = [](const char* msg) { fprintf(stderr, "ERROR: %s\n", msg); return 2; };
    if (opt.merge.enabled) {                            /* src/options.cpp:112-157 */
        if (!deviceFastq) { fprintf(stderr, "ERROR: merging mode needs --device_fastq\n"); return 2; }
        if (in2.empty() && !interleavedIn) { fprintf(stderr, "ERROR: read2 input should be specified by --in2 for merging mode\n"); return 2; }
        opt.correction.enabled = true;
        if (mergedOut.empty() && !toStdout && !out1.empty() && out2.empty()) {     /* :122-126 */
            std::cerr << "You specified --out1, but haven't specified --merged_out in merging mode. Using --out1 to store the merged reads to be compatible with fastp 0.19.8" << std::endl << std::endl;
            mergedOut = out1; out1.clear();
        }
        if (opt.merge.includeUnmerged) {
            if (!out1.empty()) { std::cerr << "You specified --include_unmerged in merging mode. Ignoring argument --out1 = " << out1 << std::endl; out1.clear(); }
            if (!out2.empty()) { std::cerr << "You specified --include_unmerged in merging mode. Ignoring argument --out2 = " << out2 << std::endl; out2.clear(); }
            if (!unpaired1.empty()) { std::cerr << "You specified --include_unmerged in merging mode. Ignoring argument --unpaired1 = " << unpaired1 << std::endl; unpaired1.clear(); }
            /* the reference names --unpaired1 here too (options.cpp:140-141) */
            if (!unpaired2.empty()) { std::cerr << "You specified --include_unmerged in merging mode. Ignoring argument --unpaired1 = " << unpaired2 << std::endl; unpaired2.clear(); }
        }
        if (mergedOut.empty() && !toStdout) return fail("In merging mode, you should either specify --merged_out or enable --stdout");
        if (!mergedOut.empty()) {
            if (mergedOut == out1 || mergedOut == out2) { fprintf(stderr, "ERROR: --merged_out and --out1 / --out2 shouldn't have same file name\n"); return 2; }
            if (mergedOut == unpaired1) return fail("--merged_out and --unpaired1 shouldn't have same file name");
            if (mergedOut == unpaired2) return fail("--merged_out and --unpaired2 shouldn't have same file name");
        }
    }
    if (toStdout) {                                      /* src/options.cpp:171-179 */
        std::cerr << "Streaming uncompressed " << (opt.merge.enabled ? "merged" : opt.paired ? "interleaved" : "") << " reads to STDOUT..." << std::endl;
        if (opt.paired && !opt.merge.enabled) std::cerr << "Enable interleaved output mode for paired-end input." << std::endl;
        std::cerr << std::endl;
    }
    if (!in2.empty() && interleavedIn) return fail("<in2> is not allowed when <in1> is specified as interleaved mode by (--interleaved_in)");
    if (!opt.paired) {                                  /* src/options.cpp:222-229 */
        if (!unpaired1.empty()) { std::cerr << "Not paired-end mode. Ignoring argument --unpaired1 = " << unpaired1 << std::endl; unpaired1.clear(); }
        if (!unpaired2.empty()) { std::cerr << "Not paired-end mode. Ignoring argument --unpaired2 = " << unpaired2 << std::endl; unpaired2.clear(); }
        if (!overlappedOut.empty()) { std::cerr << "Not paired-end mode. Ignoring argument --overlapped_out = " << overlappedOut << std::endl; overlappedOut.clear(); }   /* :230-233 */
    }
    if (!unpaired1.empty()) {                           /* src/options.cpp:240-276 */
        if (unpaired1 == out1) return fail("--unpaired1 and --out1 shouldn't have same file name");
        if (unpaired1 == out2) return fail("--unpaired1 and --out2 shouldn't have same file name");
    }
    if (!unpaired2.empty()) {
        if (unpaired2 == out1) return fail("--unpaired2 and --out1 shouldn't have same file name");
        if (unpaired2 == out2) return fail("--unpaired2 and --out2 shouldn't have same file name");
    }
    if (!failedOut.empty()) {
        if (failedOut == out1) return fail("--failed_out and --out1 shouldn't have same file name");
        if (failedOut == out2) return fail("--failed_out and --out2 shouldn't have same file name");
        if (failedOut == unpaired1) return fail("--failed_out and --unpaired1 shouldn't have same file name");
        if (failedOut == unpaired2) return fail("--failed_out and --unpaired2 shouldn't have same file name");
        if (opt.merge.enabled && failedOut == mergedOut) return fail("--failed_out and --merged_out shouldn't have same file name");
    }
    if (!indexList1.empty()) opt.indexFilter.blacklist1 = loadBarcodes(indexList1);     /* Options::initIndexFiltering (src/options.cpp:462-481) */
    if (!indexList2.empty()) opt.indexFilter.blacklist2 = loadBarcodes(indexList2);
    opt.indexFilter.enabled = !(opt.indexFilter.blacklist1.empty() && opt.indexFilter.blacklist2.empty());
    /* the writers that exist (src/peprocessor.cpp:64-72): --unpaired2 has its own only when it names another file than --unpaired1 */
    const bool unpairedLeft = !unpaired1.empty(), unpairedRight = !unpaired2.empty() && unpaired2 != unpaired1;
    std::ifstream f1, f2;
    if (!stdinInput) f1.open(in1);
    if (opt.paired && !interleavedIn) f2.open(in2);
    if ((!stdinInput && !f1) || (opt.paired && !interleavedIn && !f2)) { fprintf(stderr, "cannot open input\n"); return 1; }
    if (!deviceFastq && ((in1.size() > 3 && in1.compare(in1.size() - 3, 3, ".gz") == 0))) { fprintf(stderr, "compressed input needs --device_fastq\n"); return 2; }
    /* text path inputs: .gz / BGZF inputs are inflated on the host (fp_gz_open: zlib streaming reader, plain files and pipes pass through) */
    void* g1 = nullptr; void* g2 = nullptr;
    std::string buf1, buf2;                             /* what has been read and not yet consumed, per input */
    bool eof1 = false, eof2 = !opt.paired || interleavedIn;
    if (deviceFastq) {
        g1 = fp_gz_open(in1.c_str()); g2 = opt.paired && !interleavedIn ? fp_gz_open(in2.c_str()) : nullptr;
        if (!g1 || (opt.paired && !interleavedIn && !g2)) { fprintf(stderr, "cannot open input\n"); return 1; }
    }
    if (maxLen == 0) {                                  /* Evaluator::evaluateSeqLen peeks at the first records (src/evaluator.cpp:54-76) */
        std::vector<uint8_t> head(1 << 20);
        int64_t got;
        if (stdinInput) {                               /* a pipe is read once: the bytes peeked at start the first chunk */
            got = fp_gz_read(g1, head.data(), (int64_t)head.size());
            if (got < 0) { fprintf(stderr, "fastp_gpu_cli: corrupt compressed input\n"); return 1; }
            buf1.assign(reinterpret_cast<const char*>(head.data()), (size_t)got);
            if (got < (int64_t)head.size()) eof1 = true;
        } else {
            void* gp = fp_gz_open(in1.c_str());
            got = gp ? fp_gz_read(gp, head.data(), (int64_t)head.size()) : 0;
            fp_gz_close(gp);
        }
        maxLen = 151;
        int n = 0; size_t ls = 0;
        for (size_t i = 0; i < (size_t)std::max<int64_t>(got, 0) && n < 4000; i++)
            if (head[i] == '\n') { if (n % 4 == 1) maxLen = std::max(maxLen, (int)(i - ls)); n++; ls = i + 1; }
        maxLen += 64;
    }
    if (chunkBytes == 0) chunkBytes = (size_t)packSize * (size_t)(2 * maxLen + 64);
    GpuChainWorker worker(&opt, maxLen, 0, packSize);
    if (!worker.ok()) { fprintf(stderr, "fastp_gpu_cli: %s\n", worker.error().c_str()); return 1; }
    /* one entry per output stream, indexed like processFastqText's outs; an empty path: that writer does not exist (--overlapped_out has no
       file-name checks: the reference has none for it) */
    struct OutStream { std::string path; bool gz = false; std::ofstream file; std::string text; };
    OutStream outs[FQ_TEXT_OUTS] = {{opt.merge.enabled ? mergedOut : ""}, {out1}, {out2}, {unpaired1}, {unpairedRight ? unpaired2 : ""},
                                    {failedOut}, {overlappedOut}};
    for (OutStream& o : outs)
        if (!o.path.empty()) o.file.open(o.path);       /* every writer creates its file, even one that stays empty */
    if (deviceFastq) {
        if (opt.paired && (interleavedIn || (toStdout && !opt.merge.enabled)) && !worker.setInterleaved(interleavedIn, toStdout && !opt.merge.enabled)) {
            fprintf(stderr, "fastp_gpu_cli: interleaved text: %s\n", fp_last_error()); return 1;
        }
        if (evalDup || dedup) {                            /* accuracy level: 3 with --dedup, else 1, unless given (src/main.cpp:203-209) */
            if (!worker.setDedup(dupLevel ? dupLevel : (dedup ? 3 : 1), dedup)) { fprintf(stderr, "fastp_gpu_cli: duplicate filter: %s\n", fp_last_error()); return 1; }
        }
        if (opt.indexFilter.enabled && !worker.setIndexFilter(opt.indexFilter.blacklist1, opt.indexFilter.blacklist2, opt.indexFilter.threshold)) {
            fprintf(stderr, "fastp_gpu_cli: index filter: %s\n", fp_last_error()); return 1;
        }
        /* text path: raw file chunks go to the device, which parses, filters and re-encodes them (fp_fastq_process_host);
           whatever a chunk's last, incomplete record (or the longer side of a pair) leaves over is carried into the next chunk */
        /* .gz outputs are written as one gzip member per round, compressed by `zthreads` host threads (what the reference's writer threads do
           per pack, src/writerthread.cpp:118-168); --stdout is never compressed (src/options.cpp:171-179) and carries FASTQ only */
        auto fill = [&](void* g, std::string& buf, bool& eof) {
            if (eof) return;
            const size_t old = buf.size();
            buf.resize(old + chunkBytes);
            const int64_t got = fp_gz_read(g, reinterpret_cast<uint8_t*>(&buf[old]), (int64_t)chunkBytes);
            if (got < 0) { fprintf(stderr, "fastp_gpu_cli: corrupt compressed input\n"); exit(1); }
            buf.resize(old + (size_t)got);
            if ((size_t)got < chunkBytes) eof = true;
        };
        for (OutStream& o : outs) o.gz = o.path.size() > 3 && o.path.compare(o.path.size() - 3, 3, ".gz") == 0;
        std::vector<uint8_t> zbuf;
        auto emit = [&](OutStream& o) {
            const std::string& t = o.text;
            if (!o.file.is_open() || t.empty()) return;
            if (!o.gz) { o.file << t; return; }
            int64_t nz = 0;
            zbuf.resize((size_t)fp_gz_deflate_bound((int64_t)t.size(), 1 << 20));
            if (fp_gz_deflate(reinterpret_cast<const uint8_t*>(t.data()), (int64_t)t.size(), zbuf.data(), (int64_t)zbuf.size(), &nz, 1 << 20, zlevel, zthreads) != FP_OK) {
                fprintf(stderr, "fastp_gpu_cli: gzip output failed\n"); exit(1);
            }
            o.file.write(reinterpret_cast<const char*>(zbuf.data()), (std::streamsize)nz);
        };
        auto to_stdout = [&](const std::string& t) {
            if (!t.empty() && fwrite(t.data(), 1, t.size(), stdout) != t.size()) { fprintf(stderr, "fastp_gpu_cli: writing to STDOUT failed\n"); exit(1); }
        };
        const bool twoFiles = opt.paired && !interleavedIn;
        for (;;) {
            fill(g1, buf1, eof1);
            if (twoFiles) fill(g2, buf2, eof2);
            const bool final = eof1 && eof2;
            /* merged, out1 and out2 are always encoded; the others only for a writer that exists (it decides where a failing read goes) */
            std::string* texts[FQ_TEXT_OUTS]; size_t c1 = 0, c2 = 0; long units = 0;
            for (int s = 0; s < FQ_TEXT_OUTS; s++) {
                outs[s].text.clear();
                texts[s] = s <= FP_FQ_OUT_R2 || !outs[s].path.empty() ? &outs[s].text : nullptr;
            }
            if (!worker.processFastqText(buf1.data(), buf1.size(), buf2.data(), buf2.size(), final, phred64, texts, &c1, &c2, &units)) {
                fprintf(stderr, "fastp_gpu_cli: %s\n", worker.error().c_str()); return 1;
            }
            /* --stdout carries out1 (interleaved for pairs), or in merging mode the merged reads unless --merged_out is given (:672-678) */
            const int toOut = opt.merge.enabled ? FP_FQ_OUT_MERGED : FP_FQ_OUT_R1;
            if (toStdout && outs[toOut].path.empty()) to_stdout(outs[toOut].text);
            /* the unpaired-2 text reaches its file only when both writers exist (peprocessor.cpp:681-686) */
            for (int s = 0; s < FQ_TEXT_OUTS; s++)
                if (s != FP_FQ_OUT_UNPAIRED2 || unpairedLeft) emit(outs[s]);
            buf1.erase(0, c1); if (twoFiles) buf2.erase(0, c2);
            if (worker.inputEnded()) break;                    /* a reader gave up on a record: the reference stops reading there */
            if (final && (units == 0 || (buf1.empty() && buf2.empty()))) break;
            if (final && c1 == 0 && c2 == 0) break;
        }
        fp_gz_close(g1); fp_gz_close(g2);
        if (toStdout && (fflush(stdout) != 0 || ferror(stdout))) { fprintf(stderr, "fastp_gpu_cli: writing to STDOUT failed\n"); return 1; }
    } else
    for (;;) {
        ReadPack* lp = new ReadPack{new Read*[packSize], 0};
        ReadPack* rp = opt.paired ? new ReadPack{new Read*[packSize], 0} : nullptr;
        while (lp->count < packSize) {
            Read* a = readRecord(f1);
            if (!a) break;
            if (opt.paired) { Read* b = readRecord(f2); if (!b) { delete a; break; } rp->data[rp->count++] = b; }
            lp->data[lp->count++] = a;
        }
        const bool last = lp->count < packSize;
        std::string s1, s2;
        if (lp->count == 0) { delete[] lp->data; delete lp; if (rp) { delete[] rp->data; delete rp; } break; }
        if (opt.paired) worker.processPairEnd(lp, rp, &s1, &s2); else worker.processSingleEnd(lp, &s1);
        if (!worker.error().empty()) { fprintf(stderr, "fastp_gpu_cli: %s\n", worker.error().c_str()); return 1; }
        if (outs[FP_FQ_OUT_R1].file.is_open()) outs[FP_FQ_OUT_R1].file << s1;
        if (outs[FP_FQ_OUT_R2].file.is_open()) outs[FP_FQ_OUT_R2].file << s2;
        if (last) break;
    }
    Stats pre1, post1, pre2, post2; FilterResult fr; std::vector<long> isize;
    if (!worker.finish(&pre1, &post1, &pre2, &post2, &fr, &isize)) { fprintf(stderr, "fastp_gpu_cli: %s\n", worker.error().c_str()); return 1; }
    long dupTotal = 0, dupCount = 0;
    if (deviceFastq && (evalDup || dedup)) worker.dupTotals(&dupTotal, &dupCount);
    if (!json.empty()) {
        std::ofstream js(json);
        auto tot = [&](long Stats::*m) { return pre1.*m + (opt.paired ? pre2.*m : 0); };
        auto tota = [&](long Stats::*m) { return post1.*m + (opt.paired ? post2.*m : 0); };
        js << "{\n \"before_filtering\": {\"total_reads\": " << tot(&Stats::mReads) << ", \"total_bases\": " << tot(&Stats::mBases)
           << ", \"q20_bases\": " << tot(&Stats::mQ20Total) << ", \"q30_bases\": " << tot(&Stats::mQ30Total) << "},\n"
           << " \"after_filtering\": {\"total_reads\": " << tota(&Stats::mReads) << ", \"total_bases\": " << tota(&Stats::mBases)
           << ", \"q20_bases\": " << tota(&Stats::mQ20Total) << ", \"q30_bases\": " << tota(&Stats::mQ30Total) << "},\n"
           << " \"filtering_result\": {\"passed_filter_reads\": " << fr.mFilterReadStats[FP_PASS_FILTER] << ", \"low_quality_reads\": " << fr.mFilterReadStats[FP_FAIL_QUALITY]
           << ", \"too_many_N_reads\": " << fr.mFilterReadStats[FP_FAIL_N_BASE] << ", \"too_short_reads\": " << fr.mFilterReadStats[FP_FAIL_LENGTH]
           << ", \"too_long_reads\": " << fr.mFilterReadStats[FP_FAIL_TOO_LONG] << ", \"low_complexity_reads\": " << fr.mFilterReadStats[FP_FAIL_COMPLEXITY]
           << ", \"adapter_dimer_reads\": " << fr.mFilterReadStats[FP_FAIL_ADAPTER_DIMER] << "},\n"
           << " \"adapter_cutting\": {\"adapter_trimmed_reads\": " << fr.mTrimmedAdapterRead << ", \"adapter_trimmed_bases\": " << fr.mTrimmedAdapterBases << "},\n"
           << " \"duplication\": {\"total\": " << dupTotal << ", \"duplicates\": " << dupCount << "},\n"
           << " \"corrected_reads\": " << fr.mCorrectedReads << ",\n \"insert_size_unknown\": " << (isize.empty() ? 0 : isize.back()) << "\n}\n";
    }
    return 0;
}
