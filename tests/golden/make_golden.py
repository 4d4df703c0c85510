"""Generates tests/golden/*.npz from the reference's own test fixtures.

Needs a checkout of featureform/embeddinghub:
    python tests/golden/make_golden.py <reference checkout>
Sources:
  provider/test_files/embeddings.csv         (5 x 768 f32, provider/vectorstore_test.go:172-211)
  provider/vectorstore_test.go:214-226       (768-d search vector)
The values are parsed exactly as the Go test does (strconv.ParseFloat(.., 32)).
"""
import csv
import os
import re
import sys

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    ref = os.path.join(sys.argv[1], "provider")
    ents, vecs = [], []
    with open(os.path.join(ref, "test_files/embeddings.csv")) as f:
        r = csv.reader(f)
        next(r)
        for row in r:
            ents.append(row[0])
            vecs.append(np.array([np.float32(float(x)) for x in row[1].split(",")], np.float32))
    src = open(os.path.join(ref, "vectorstore_test.go")).read()
    m = re.search(r'func getSearchVector.*?vectorStr := "([^"]+)"', src, re.S)
    q = np.array([np.float32(float(x)) for x in m.group(1).split(",")], np.float32)
    vecs = np.stack(vecs)
    assert vecs.shape == (5, 768) and q.shape == (768,)
    np.savez(os.path.join(OUT, "vectorstore_fixture.npz"), entities=np.array(ents), vectors=vecs, query=q)
    print("wrote", vecs.shape, q.shape, ents)


if __name__ == "__main__":
    main()
