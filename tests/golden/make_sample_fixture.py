"""Makes tests/golden/sample_data/ from the reference's bundled sample_data.tgz (BASELINE.json configs[0]: 15 transcripts,
10 000 simulated 2x50 bp pairs whose names carry the truth, `@<i>:<transcript>:<position>:<fragment length>`).
Needs a salmon source tree; the outputs are committed, so the tests do not.
usage: python tests/golden/make_sample_fixture.py <salmon source tree>/sample_data.tgz"""
import gzip
import io
import os
import sys
import tarfile

src = sys.argv[1]
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sample_data")
os.makedirs(out, exist_ok=True)
with tarfile.open(src) as tf:
    for member, name in (("sample_data/transcripts.fasta", "transcripts.fasta.gz"), ("sample_data/reads_1.fastq", "reads_1.fastq.gz"),
                         ("sample_data/reads_2.fastq", "reads_2.fastq.gz")):
        data = tf.extractfile(member).read()
        with open(os.path.join(out, name), "wb") as f:
            with gzip.GzipFile(filename="", mode="wb", fileobj=f, mtime=0, compresslevel=9) as g:
                g.write(data)
        print(name, len(data), "->", os.path.getsize(os.path.join(out, name)))
