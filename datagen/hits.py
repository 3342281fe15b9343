"""Synthetic ClickBench `hits` table (BASELINE.json configs[4]).

The real hits.parquet (100 M rows, 105 columns) is not in this image and the reference pins ClickBench plans on an EMPTY
table only (python/pysail/tests/spark/test_clickbench.py:122-140), so there is no reference result to reproduce: this
generator makes a table with the columns the 43 queries touch (names, order and integer widths of the reference's schema,
test_clickbench.py:11-119) and with the skew the queries are about -- a Zipf-distributed UserID / URL / SearchPhrase
vocabulary, ~70 % empty search phrases, a dominant CounterID 62, July 2013 dates.  Differences from the reference's view,
stated once: strings are Utf8View (the reference reads the file's BINARY columns; DataFusion runners set
`binary_as_string`), EventDate is Date32 (the reference's view does `date_add('1970-01-01', EventDate)`,
test_clickbench.py:135) and EventTime stays Int64 seconds (the reference casts it to Timestamp; ordering by it is the same).

Deterministic for (n, seed); built by numpy column-wise, strings as views over a shared vocabulary heap.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

from .tpch import date32, strings_from_codes

COLUMNS = ["WatchID", "Title", "EventTime", "EventDate", "CounterID", "ClientIP", "RegionID", "UserID", "URL", "Referer", "IsRefresh",
           "ResolutionWidth", "MobilePhone", "MobilePhoneModel", "TraficSourceID", "SearchEngineID", "SearchPhrase", "AdvEngineID",
           "WindowClientWidth", "WindowClientHeight", "IsLink", "IsDownload", "DontCountHits", "RefererHash", "URLHash"]

DOMAINS = ["yandex.ru", "www.google.com", "mail.ru", "vk.com", "avito.ru", "news.google.ru", "auto.ru", "kinopoisk.ru", "rambler.ru",
           "market.yandex.ru", "maps.google.com", "livejournal.com", "ok.ru", "wikipedia.org", "hh.ru", "drom.ru", "e1.ru", "irr.ru"]
WORDS = ["купить", "цена", "погода", "фото", "новости", "игры", "онлайн", "скачать", "смотреть", "фильм", "авто", "работа", "карта",
         "недвижимость", "отзывы", "google", "Google", "maps", "video", "mail", "search", "top", "free", "best", "2013", "москва", "спб"]
MODELS = ["iPhone", "iPad", "GT-I9300", "Lumia 920", "Nexus 4", "Xperia Z", "GT-N7100", "One X", "Desire", "Galaxy Tab", "iPod", "E71"]
WIDTHS = np.array([0, 320, 768, 1024, 1280, 1366, 1440, 1536, 1600, 1680, 1920, 2560], dtype=np.int16)


def zipf_codes(rng, n: int, vocab: int, a: float = 1.15) -> np.ndarray:
    """n draws from {0..vocab-1} with P(k) ~ 1/(k+1)^a: a few hot values and a long tail, like user / URL ids in a web log"""
    w = 1.0 / np.power(np.arange(1, vocab + 1, dtype=np.float64), a)
    cdf = np.cumsum(w)
    cdf /= cdf[-1]
    return np.searchsorted(cdf, rng.random(n), side="right").astype(np.int64).clip(0, vocab - 1)


def phrase_vocab(rng, k: int, lo: int, hi: int) -> list:
    out, seen = [], set()
    while len(out) < k:
        s = " ".join(WORDS[i] for i in rng.integers(0, len(WORDS), int(rng.integers(lo, hi + 1))))
        if s not in seen:
            seen.add(s)
            out.append(s)
    return out


def url_vocab(rng, k: int) -> list:
    out = []
    for i in range(k):
        d = DOMAINS[int(rng.integers(0, len(DOMAINS)))]
        path = "/".join(WORDS[j] for j in rng.integers(0, len(WORDS), int(rng.integers(1, 4))))
        out.append(f"http://{d}/{path}/{i}" + ("?q=" + WORDS[int(rng.integers(0, len(WORDS)))] if i % 3 == 0 else ""))
    return out


def vocab_hash(k: int, salt: int) -> np.ndarray:
    """a 64-bit hash per vocabulary entry (stands in for the URLHash / RefererHash columns the source computes upstream):
    splitmix64 of the entry's index"""
    z = (np.arange(k, dtype=np.uint64) + np.uint64(salt)) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return (z ^ (z >> np.uint64(31))).view(np.int64)


def hits(n: int, seed: int = 0, strings: str = "view", columns=None) -> pa.Table:
    rng = np.random.default_rng(seed)
    n_users = max(8, n // 6)
    n_urls = min(max(16, n // 10), 200_000)       # string vocabularies are capped: they are built by Python loops
    n_refs = min(max(8, n // 20), 100_000)
    n_phr = min(max(8, n // 50), 50_000)
    n_titles = min(max(8, n // 25), 100_000)

    users = rng.integers(1 << 40, 1 << 62, n_users, dtype=np.int64)
    urls = [""] + url_vocab(rng, n_urls)
    refs = [""] + url_vocab(rng, n_refs)
    phrases = [""] + phrase_vocab(rng, n_phr, 1, 4)
    titles = [""] + phrase_vocab(rng, n_titles, 2, 6)
    models = [""] + MODELS

    day = rng.integers(0, 31, n)                                        # 2013-07-01 .. 2013-07-31
    date0 = 15887                                                       # days since the epoch of 2013-07-01
    url_c = np.where(rng.random(n) < 0.01, 0, 1 + zipf_codes(rng, n, n_urls))
    ref_c = np.where(rng.random(n) < 0.30, 0, 1 + zipf_codes(rng, n, n_refs))
    phr_c = np.where(rng.random(n) < 0.70, 0, 1 + zipf_codes(rng, n, n_phr))
    ttl_c = np.where(rng.random(n) < 0.05, 0, 1 + zipf_codes(rng, n, n_titles))
    mdl_c = np.where(rng.random(n) < 0.90, 0, 1 + zipf_codes(rng, n, len(MODELS), 1.0))
    counter = np.where(rng.random(n) < 0.06, 62, 1 + zipf_codes(rng, n, max(4, n // 200))).astype(np.int32)
    url_hash, ref_hash = vocab_hash(len(urls), 1), vocab_hash(len(refs), 2)

    cols = {
        "WatchID": rng.permutation(n).astype(np.int64) * 0x9E3779B1 + (1 << 50),
        "Title": (ttl_c, titles),
        "EventTime": ((date0 + day) * 86400 + rng.integers(0, 86400, n)).astype(np.int64),
        "EventDate": date32((date0 + day).astype(np.int32)),
        "CounterID": counter,
        "ClientIP": rng.integers(-(1 << 31), 1 << 31, max(4, n // 8), dtype=np.int64).astype(np.int32)[zipf_codes(rng, n, max(4, n // 8), 1.05)],
        "RegionID": zipf_codes(rng, n, 5000, 1.2).astype(np.int32),
        "UserID": users[zipf_codes(rng, n, n_users)],
        "URL": (url_c, urls),
        "Referer": (ref_c, refs),
        "IsRefresh": (rng.random(n) < 0.10).astype(np.int16),
        "ResolutionWidth": WIDTHS[rng.integers(0, len(WIDTHS), n)],
        "MobilePhone": np.where(mdl_c == 0, 0, rng.integers(1, 200, n)).astype(np.int16),
        "MobilePhoneModel": (mdl_c, models),
        "TraficSourceID": rng.integers(-1, 10, n).astype(np.int16),
        "SearchEngineID": np.where(rng.random(n) < 0.5, 0, rng.integers(1, 90, n)).astype(np.int16),
        "SearchPhrase": (phr_c, phrases),
        "AdvEngineID": np.where(rng.random(n) < 0.95, 0, rng.integers(1, 60, n)).astype(np.int16),
        "WindowClientWidth": WIDTHS[rng.integers(0, len(WIDTHS), n)],
        "WindowClientHeight": (WIDTHS[rng.integers(0, len(WIDTHS), n)] // 2).astype(np.int16),
        "IsLink": (rng.random(n) < 0.15).astype(np.int16),
        "IsDownload": (rng.random(n) < 0.02).astype(np.int16),
        "DontCountHits": (rng.random(n) < 0.08).astype(np.int16),
        "RefererHash": ref_hash[ref_c],
        "URLHash": url_hash[url_c],
    }
    names = list(columns) if columns is not None else COLUMNS
    arrays = []
    for c in names:
        v = cols[c]
        if isinstance(v, tuple):
            arrays.append(strings_from_codes(np.asarray(v[0], dtype=np.int64), v[1], "view" if strings == "view" else "utf8"))
        elif isinstance(v, pa.Array):
            arrays.append(v)
        else:
            arrays.append(pa.array(np.ascontiguousarray(v)))
    return pa.table(arrays, names=names)


def stored(table: pa.Table) -> pa.Table:
    """`hits(n)` with the column types the reference's hits.parquet stores (test_clickbench.py:11-119): strings as `binary`
    (Parquet BYTE_ARRAY without a UTF8 annotation) and EventDate as UInt16 days since the epoch (INT32 annotated INT(16, unsigned));
    the Int16 / Int32 / Int64 columns are stored as they are.  sail_b200.clickbench.view turns the stored types back into `hits`'s."""
    arrays = []
    for f, c in zip(table.schema, table.columns):
        if pa.types.is_string_view(f.type) or pa.types.is_string(f.type):
            c = c.cast(pa.binary())
        elif pa.types.is_date32(f.type):
            c = c.cast(pa.int32()).cast(pa.uint16())
        arrays.append(c)
    return pa.table(arrays, names=table.schema.names)


def delta_encoding(schema: pa.Schema) -> dict:
    """pyarrow `column_encoding` for a stored hits table written without dictionaries: integer and timestamp columns as
    DELTA_BINARY_PACKED, strings as DELTA_BYTE_ARRAY -- the encodings a Parquet V2 writer falls back to when a column outgrows
    its dictionary.  Write it with `use_dictionary=False, data_page_version="2.0"`."""
    enc = {}
    for f in schema:
        if pa.types.is_integer(f.type) or pa.types.is_timestamp(f.type):
            enc[f.name] = "DELTA_BINARY_PACKED"
        elif pa.types.is_binary(f.type) or pa.types.is_string(f.type):
            enc[f.name] = "DELTA_BYTE_ARRAY"
    return enc
