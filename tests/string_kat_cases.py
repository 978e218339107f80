"""Known-answer vectors of the reference's Utf8 expressions, each cited by file:line of the reference tree
(datafusion-ext-exprs/src/*.rs, datafusion-ext-commons/src/arrow/cast.rs).

Every case is (id, column values, expression kind, pattern, scalar operand or None, expected).  A scalar operand means the
reference evaluated the expression over a Utf8 literal (`phys_expr::lit`) instead of the column; the result is that literal's
answer on every row."""

STRING_MATCH_KATS = [
    # string_starts_with.rs:132-166 test_ok
    ("starts_with_test_ok", [None, "rabaok", "rraara", "s_skdo[]ra.,?';,{}\ra", " raefuwidn"], "StartsWith", "ra", None,
     [None, True, False, False, False]),
    # string_starts_with.rs:168-197 test_scalar_string
    ("starts_with_test_scalar_string", ["Hello, Rust", "Hello, He", None, "RustHe", "HellHe"], "StartsWith", "ra", "rarrr",
     [True, True, True, True, True]),
    # string_ends_with.rs:133-170 test_array
    ("ends_with_test_array", ["abrrbrr", "rrjndebcsabdji", None, "rr", "roser r"], "EndsWith", "rr", None,
     [True, False, None, True, False]),
    # string_ends_with.rs:172-211 test_scalar_string
    ("ends_with_test_scalar_string", ["Hello, Rust", "Hello, He", None, "RustHe", "HellHe"], "EndsWith", "He", "Hello, Rust",
     [False, False, False, False, False]),
    # string_contains.rs:130-169 test_ok
    ("contains_test_ok", ["abrr", "barr", "rnba", "nbar", None], "Contains", "ba", None,
     [False, True, True, True, None]),
    # string_contains.rs:171-207 test_scalar_string
    ("contains_test_scalar_string", ["abrr", "barr", "rnba", "nbar", None], "Contains", "ba", "abab",
     [True, True, True, True, True]),
]

# cast.rs:576-599 test_string_to_bigint: (input, expected) of cast(Utf8 -> Int64)
STRING_TO_BIGINT_KAT = [
    (None, None), ("123", 123), ("987", 987), ("987.654", 987), ("123456789012345", 123456789012345),
    ("-123456789012345", -123456789012345), ("999999999999999999999999999999999", None),
]

# the edge cases the toLong port accepts or refuses (cast.rs:287-361), per target width in bits: (input, bits, expected)
TO_LONG_EDGE_CASES = [
    ("", 64, None), ("-", 64, None), ("+", 64, None), (".", 64, 0), ("-.", 64, 0), ("+.", 64, 0), ("1.", 64, 1), ("-1.", 64, -1),
    ("1.2x", 64, None), ("1.25", 64, 1), (" 1", 64, None), ("1 ", 64, None), ("+7", 64, 7), ("--1", 64, None), ("1e3", 64, None),
    ("0x10", 64, None), ("007", 64, 7), ("-0", 64, 0), ("..", 64, None), ("1..", 64, None), ("１", 64, None),
    ("127", 8, 127), ("128", 8, None), ("-128", 8, -128), ("-129", 8, None),
    ("32767", 16, 32767), ("32768", 16, None), ("-32768", 16, -32768), ("-32769", 16, None),
    ("2147483647", 32, 2147483647), ("2147483648", 32, None), ("-2147483648", 32, -2147483648), ("-2147483649", 32, None),
    ("9223372036854775807", 64, 9223372036854775807), ("9223372036854775808", 64, None),
    ("-9223372036854775808", 64, -9223372036854775808), ("-9223372036854775809", 64, None),
    ("-9223372036854775808.999", 64, -9223372036854775808), ("99999999999999999999", 64, None),
]
