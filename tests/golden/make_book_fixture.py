#!/usr/bin/env python3
"""Extract the 18-book library of the reference's faceting tests into a fixture.

Source : src/Infidex.Tests/FacetingTests.cs of the reference repository, CreateBookLibrary() (:589-641): CreateBookDoc(id, title, author, year,
         genre, description) -> fields title (High, indexable), author (Med, indexable, facetable), year (Low, not indexable,
         facetable), genre (Low, indexable, facetable), description (Med, indexable) (:643-676).
Output : tests/golden/books.json  (list of [id, title, author, year, genre, description])
Usage  : make_book_fixture.py <path to FacetingTests.cs>; the output is committed, so the tests never read the reference.
"""
import json, os, re, sys
src = sys.argv[1]
text = open(src, encoding="utf-8-sig").read()
body = text[text.index("private static Document[] CreateBookLibrary()"):text.index("private static Document CreateBookDoc(")]
STR = r'"((?:[^"\\]|\\.)*)"'
pat = re.compile(r"CreateBookDoc\(\s*(\d+)L\s*,\s*" + r"\s*,\s*".join([STR] * 5) + r"\s*\)", re.S)
books = [[int(m.group(1))] + [bytes(g, "utf-8").decode("unicode_escape").encode("latin-1").decode("utf-8") if "\\" in g else g for g in m.groups()[1:]] for m in pat.finditer(body)]
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "books.json")
json.dump(books, open(out, "w", encoding="utf-8"), ensure_ascii=False, indent=0)
print(len(books), "books ->", out)
