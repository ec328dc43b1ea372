#!/usr/bin/env python3
"""Extract the `title` column of the reference's test corpus into a compact fixture.

Source : src/Infidex.Tests/movies.csv of the reference repository (40 837 rows; doc key = row index, as in
         MovieSearchParityTests.cs:1186-1204 `new Document((long)i, m.Title)`).
Output : tests/golden/movies_titles.txt.gz  (one title per line; titles containing newlines are kept with \\n escaped)
Usage  : make_movie_fixture.py <path to movies.csv>; the output is committed, so the tests never read the reference.
"""
import csv, gzip, os, sys
src = sys.argv[1]
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "movies_titles.txt.gz")
with open(src, newline="", encoding="utf-8-sig") as f:
    rows = list(csv.DictReader(f))
titles = [r["title"] for r in rows]
with gzip.open(out, "wt", encoding="utf-8", compresslevel=9) as g:
    for t in titles:
        g.write(t.replace("\\", "\\\\").replace("\n", "\\n") + "\n")
print(len(titles), "titles ->", out, os.path.getsize(out), "bytes")
