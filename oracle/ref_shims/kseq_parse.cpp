// oracle/ref_shims/kseq_parse.cpp -- TEST INFRASTRUCTURE.  Glue around the FASTA/FASTQ parser the reference tree
// vendors (include/kseq++.hpp, klibpp::KStream -- the parser behind salmon's read files): every record's sequence line,
// as that parser delivers it.  Compiled by oracle/build_ref.sh against the header where it lies in a salmon source tree.
#include <zlib.h>

#include <kseq++.hpp>

// pass seq_out == NULL to count: returns the number of records, *total_bytes = the sum of the sequence lengths
extern "C" long ref_kseq_parse(const char* path, unsigned char* seq_out, unsigned long seq_cap, unsigned* lens_out,
                               unsigned long max_rec, unsigned long* total_bytes) {
  gzFile fp = gzopen(path, "r");
  if (!fp) return -1;
  auto ks = klibpp::make_ikstream(fp, gzread);
  klibpp::KSeq rec;
  unsigned long n = 0, tot = 0;
  while (ks >> rec) {
    if (seq_out) {
      if (n >= max_rec || tot + rec.seq.size() > seq_cap) { gzclose(fp); return -2; }
      memcpy(seq_out + tot, rec.seq.data(), rec.seq.size());
      lens_out[n] = (unsigned)rec.seq.size();
    }
    tot += rec.seq.size();
    ++n;
  }
  gzclose(fp);
  if (total_bytes) *total_bytes = tot;
  return (long)n;
}
