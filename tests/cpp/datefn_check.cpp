// datefn_check.cpp — the library's date functions (csrc/datetime.h: dt_date_fn after the argument's family cast, as OP_DATEFN runs
// them) against the tests' restatement of the reference (tests/cpp/date_fn_oracle.c), for every function and mode over:
//   every day 0000-01-01 .. 9999-12-31 (as DATE, and as DATETIME at 23:59:58); day 0, month 0 and days 29-31 of every month of a
//   leap and a non-leap year; the zero date; both sides of every midnight (+08) of the TIMESTAMP range; a sweep of TIME values.
// Prints "datefn_check ok <count>" or the first mismatches.
#include <stdio.h>
#include <string.h>
#include <vector>
#include "datetime.h"

extern "C" int64_t bk_oracle_date_fn(const char* fn, int arg, int prim, uint64_t image, int prim2, uint64_t image2, int* is_null);

using namespace bk;

struct Fn { const char* name; int id; int arg_prim; int n_args; };   // n_args: how many mode / unit values to try
static const Fn FNS[] = {
    {"year", DF_YEAR, BK_DATETIME, 1}, {"month", DF_MONTH, BK_DATETIME, 1}, {"day", DF_DAY, BK_DATETIME, 1}, {"dayofmonth", DF_DAY, BK_DATETIME, 1},
    {"quarter", DF_QUARTER, BK_DATE, 1}, {"hour", DF_HOUR, BK_TIME, 1}, {"minute", DF_MINUTE, BK_TIME, 1}, {"second", DF_SECOND, BK_TIME, 1},
    {"dayofweek", DF_DAYOFWEEK, BK_DATETIME, 1}, {"weekday", DF_WEEKDAY, BK_DATETIME, 1}, {"dayofyear", DF_DAYOFYEAR, BK_DATETIME, 1},
    {"week", DF_WEEK, BK_DATETIME, 9}, {"yearweek", DF_YEARWEEK, BK_DATETIME, 9}, {"weekofyear", DF_WEEKOFYEAR, BK_DATETIME, 1},
    {"to_days", DF_TO_DAYS, BK_TIMESTAMP, 1}, {"to_seconds", DF_TO_SECONDS, BK_TIMESTAMP, 1}, {"unix_timestamp", DF_UNIX_TIMESTAMP, BK_TIMESTAMP, 1},
    {"datediff", DF_DATEDIFF, BK_DATE, 1}, {"extract", DF_EXTRACT, BK_TIMESTAMP, 7}, {"date", DF_DATE, BK_DATETIME, 1}};

static long long checked = 0, bad = 0;

static void check(const Fn& f, int prim, uint64_t v) {
    if (prim == BK_TIME && f.arg_prim != BK_TIME) return;   // (refused when a plan is compiled)
    for (int k = 0; k < f.n_args; k++) {
        // week / yearweek: k = 0 is "no mode", then modes 0..7; extract: units 0..5, then an unknown unit
        const int oarg = f.id == DF_WEEK || f.id == DF_YEARWEEK ? k - 1 : k;
        const int larg = f.id == DF_WEEK || f.id == DF_YEARWEEK ? (k == 0 ? DT_NO_MODE : k - 1) : (f.id == DF_EXTRACT ? (k < 6 ? k : 0xFF) : 0);
        // datediff: the value against itself shifted, and against the fixed date 1995-01-01
        const uint64_t other = (uint64_t)((1995 * 13 + 1) << 5 | 1);
        uint64_t x = prim == f.arg_prim ? v : dt_family_cast(v, prim, f.arg_prim), x2 = 0;
        if (f.id == DF_DATEDIFF) { x = dt_family_cast(x, BK_DATE, BK_TIMESTAMP); x2 = dt_family_cast(other, BK_DATE, BK_TIMESTAMP); }
        const uint64_t got = dt_date_fn(f.id, larg, x, x2);
        int onull = 0;
        const int64_t want = bk_oracle_date_fn(f.name, oarg, prim, v, BK_DATE, other, &onull);
        checked++;
        const bool ok = onull ? got == DT_FN_NULL : (got != DT_FN_NULL && got == (uint64_t)want);
        if (!ok && bad++ < 20)
            printf("MISMATCH %s arg=%d prim=%d image=0x%llx: library %s0x%llx, oracle %s%lld\n", f.name, oarg, prim, (unsigned long long)v,
                   got == DT_FN_NULL ? "NULL " : "", (unsigned long long)got, onull ? "NULL " : "", (long long)want);
    }
}
static void all(int prim, uint64_t v) { for (const Fn& f : FNS) check(f, prim, v); }

int main() {
    // every calendar day, as DATE and as DATETIME late in the day
    for (int64_t y = 0; y <= 9999; y++)
        for (int64_t m = 1; m <= 12; m++) {
            const int64_t last = m == 2 ? (dt_leap(y) ? 29 : 28) : (m == 4 || m == 6 || m == 9 || m == 11 ? 30 : 31);
            for (int64_t d = 1; d <= last; d++) {
                const uint64_t date = (uint64_t)((y * 13 + m) << 5 | d);
                all(BK_DATE, date);
                all(BK_DATETIME, dt_make((uint64_t)y, (uint64_t)m, (uint64_t)d, 23, 59, 58, 0));
            }
        }
    // day 0, month 0, days 29-31 of every month (invalid ones included) of a leap and a non-leap year, and the edges of boost's range
    for (int64_t y : {2023, 2024, 1399, 1400, 1900, 2000, 9999, 10000}) {
        for (int64_t m = 0; m <= 12; m++)
            for (int64_t d : {0, 1, 28, 29, 30, 31}) {
                all(BK_DATE, (uint64_t)((y * 13 + m) << 5 | d));
                all(BK_DATETIME, dt_make((uint64_t)y, (uint64_t)m, (uint64_t)d, 7, 59, 59, 0));
            }
    }
    all(BK_DATE, 0);
    all(BK_DATETIME, 0);
    all(BK_TIMESTAMP, 0);
    // both sides of every midnight at +08 of the TIMESTAMP range
    for (int64_t day = 0; day <= (int64_t)(0xFFFFFFFFull / 86400); day++)
        for (int64_t off : {57599, 57600, 0, 1}) {
            const int64_t t = day * 86400 + off;
            if (t >= 0 && t <= 0xFFFFFFFFll) all(BK_TIMESTAMP, (uint64_t)t);
        }
    all(BK_TIMESTAMP, 0xFFFFFFFFull);
    // TIME values, negative ones included: hours up to 1023 and beyond the field, minutes and seconds over their whole 6 bits
    for (int64_t h = 0; h < 1100; h += 7)
        for (int64_t mi = 0; mi < 64; mi += 5)
            for (int64_t s = 0; s < 64; s += 9) {
                const int32_t t = (int32_t)(h << 12 | mi << 6 | s);
                all(BK_TIME, (uint64_t)(int64_t)t);
                all(BK_TIME, (uint64_t)(int64_t)-t);
            }
    if (bad) { printf("datefn_check: %lld of %lld differ\n", bad, checked); return 1; }
    printf("datefn_check ok %lld\n", checked);
    return 0;
}
