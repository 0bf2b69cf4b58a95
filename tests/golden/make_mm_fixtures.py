"""Copies the reference's MatrixMarket TEST DATA (not code) into tests/golden/matrix_market/.
Source: sprs/data/matrix_market/ of a sprs checkout -- the files the reference's io.rs tests
read (io.rs:476-800).  Only the real / integer files the f64 path can meet are kept.
Run:  python tests/golden/make_mm_fixtures.py <path to a sprs checkout>"""
import os
import shutil
import sys

DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "matrix_market")
FILES = ["simple.mm", "simple_int.mm", "symmetric.mm", "pattern.mm",
         "bad_files/not_enough_entries.mm", "bad_files/too_many_elems_in_entry.mm",
         "complex/simple.mtx", "complex/hermitian-int.mtx"]

if __name__ == "__main__":
    src = os.path.join(sys.argv[1], "sprs", "data", "matrix_market")
    for f in FILES:
        dst = os.path.join(DST, f)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(os.path.join(src, f), dst)
        print("copied", f)
