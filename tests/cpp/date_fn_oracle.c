/* date_fn_oracle.c — the reference's date-part and day-number functions restated for the tests, independently of csrc/datetime.h:
 * the reference's own civil-date form (days_from_civil / localtime_fixed_r, src/common/datetime.cpp:24-98), the boost::gregorian
 * rules the reference relies on written out as plain loops and tables, and the functions of src/expr/internal_functions.cpp one by one.
 * Test infrastructure only: tests/test_date_fn.py checks it against the reference's known answers (tests/golden/date_fn_vectors.json),
 * tests/cpp/datefn_check.cpp compares the library's datetime.h with it, and the GPU tests compute their expected columns with it. */
#include <stdint.h>
#include <string.h>

enum { P_DATETIME = 14, P_TIMESTAMP = 15, P_DATE = 16, P_TIME = 18 };   /* pb::PrimitiveType (include/bkgpu_plan.h) */

/* ---- ExprValue::cast_to inside the date/time family (expr_value.h:534-573; datetime.cpp) ---- */
static int64_t div_floor(int64_t a, int64_t b) { return (a >= 0 ? a : a - b + 1) / b; }
static int64_t days_from_civil(int64_t y, int64_t m, int64_t d) {                               /* datetime.cpp:31-38 */
    y -= m <= 2;
    const int64_t era = div_floor(y, 400), yoe = y - era * 400;
    const int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1, doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}
typedef struct { int64_t year, month, day, hour, minute, second; } Civil;
static Civil localtime_fixed(int64_t t) {                                                       /* datetime.cpp:54-98, UTC+8 */
    Civil c;
    t += 8 * 3600;
    int64_t days = t / 86400, rem = t % 86400;
    if (rem < 0) { rem += 86400; days--; }
    const int64_t z = days + 719468, era = div_floor(z, 146097), doe = z - era * 146097;
    const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365, doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const int64_t mp = (5 * doy + 2) / 153;
    c.day = doy - (153 * mp + 2) / 5 + 1;
    c.month = mp < 10 ? mp + 3 : mp - 9;
    c.year = yoe + era * 400 + (c.month <= 2);
    c.hour = rem / 3600; c.minute = rem % 3600 / 60; c.second = rem % 60;
    return c;
}
static uint64_t make_dt(uint64_t y, uint64_t mo, uint64_t d, uint64_t h, uint64_t mi, uint64_t s) {   /* datetime.h:28-33 */
    return ((y * 13 + mo) << 46) | (d << 41) | (h << 36) | (mi << 30) | (s << 24);
}
static int64_t dt_year(uint64_t dt) { return (int64_t)(((dt >> 46) & 0x1FFFF) / 13); }             /* datetime.h:35-43 */
static int64_t dt_month(uint64_t dt) { return (int64_t)(((dt >> 46) & 0x1FFFF) % 13); }
static int64_t dt_day(uint64_t dt) { return (int64_t)((dt >> 41) & 0x1F); }
static uint32_t datetime_to_timestamp(uint64_t dt) {                                            /* datetime.cpp:304-331 */
    if (dt == 0 || dt_month(dt) == 0 || dt_day(dt) == 0) return 0;
    const int64_t t = days_from_civil(dt_year(dt), dt_month(dt), dt_day(dt)) * 86400 + (int64_t)((dt >> 36) & 0x1F) * 3600 +
                      (int64_t)((dt >> 30) & 0x3F) * 60 + (int64_t)((dt >> 24) & 0x3F) - 8 * 3600;
    return t <= 0 ? 0 : (uint32_t)t;
}
static uint64_t timestamp_to_datetime(uint32_t ts) {                                            /* datetime.cpp:352-373 */
    if (ts == 0) return 0;
    const Civil c = localtime_fixed(ts);
    return make_dt((uint64_t)c.year, (uint64_t)c.month, (uint64_t)c.day, (uint64_t)c.hour, (uint64_t)c.minute, (uint64_t)c.second);
}
static uint64_t to_datetime(int prim, uint64_t v) {
    if (prim == P_DATETIME) return v;
    if (prim == P_TIMESTAMP) return timestamp_to_datetime((uint32_t)v);
    return (uint64_t)(uint32_t)v << 41;                                                          /* DATE: date_to_datetime */
}
static uint64_t cast_to(int from, uint64_t v, int to) {                                         /* (TIME sources are not given) */
    if (from == to) return v;
    const uint64_t dt = to_datetime(from, v);
    if (to == P_DATETIME) return dt;
    if (to == P_TIMESTAMP) return datetime_to_timestamp(dt);
    if (to == P_DATE) return (dt >> 41) & 0x3FFFFF;
    return (uint64_t)(int64_t)(int32_t)(((dt >> 24) & 0x3F) | (((dt >> 30) & 0x3F) << 6) | (((dt >> 36) & 0x1F) << 12));   /* TIME */
}

/* ---- boost::gregorian: the date constructor's checks, day_of_week, day_of_year, week_number ---- */
static int is_leap(int64_t y) { return y % 4 == 0 && (y % 100 != 0 || y % 400 == 0); }
static int month_len(int64_t y, int64_t m) {
    static const int len[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    return m == 2 && is_leap(y) ? 29 : len[m - 1];
}
static int greg_ok(int64_t y, int64_t m, int64_t d) { return y >= 1400 && y <= 9999 && m >= 1 && m <= 12 && d >= 1 && d <= month_len(y, m); }
static int64_t day_of_week(int64_t y, int64_t m, int64_t d) { int64_t w = (days_from_civil(y, m, d) + 4) % 7; return w < 0 ? w + 7 : w; }   /* 0 = Sunday */
static int64_t day_of_year(int64_t y, int64_t m, int64_t d) {
    int64_t n = d;
    for (int64_t k = 1; k < m; k++) n += month_len(y, k);
    return n;
}
static int64_t iso_week(int64_t y, int64_t m, int64_t d) {
    /* ISO 8601: the week (Monday..Sunday) that holds the year's first Thursday is week 1; a date in the days before it belongs
       to the last week of the year before, a date after the last such week to week 1 of the year after */
    const int64_t day = days_from_civil(y, m, d);
    int64_t wk_year = y + 1;
    for (;;) {
        const int64_t jan1 = days_from_civil(wk_year, 1, 1);
        const int64_t first_thursday = jan1 + (4 - day_of_week(wk_year, 1, 1) + 7) % 7;
        const int64_t week1_monday = first_thursday - 3;
        if (day >= week1_monday) return (day - week1_monday) / 7 + 1;
        wk_year--;
    }
}
/* calc_mode + calc_week (internal_functions.cpp:1905-2026) */
static void calc_mode(int mode, int* monday_first, int* zero_range, int* with_4_days) {
    static const int table[8][3] = {{0, 1, 0}, {1, 1, 1}, {0, 0, 0}, {1, 0, 1}, {0, 1, 1}, {1, 1, 0}, {0, 0, 1}, {1, 0, 0}};
    *monday_first = table[mode][0]; *zero_range = table[mode][1]; *with_4_days = table[mode][2];
}
static int calc_week(uint64_t dt, int mode, int is_yearweek, int64_t* year, int64_t* weeks) {
    *year = dt_year(dt);
    const int64_t month = dt_month(dt), day = dt_day(dt);
    if (month == 0 || day == 0) return -1;
    if (!greg_ok(*year, 1, 1) || !greg_ok(*year, month, day)) return -1;
    int64_t doy = day_of_year(*year, month, day), first = day_of_week(*year, 1, 1);
    int monday_first = 0, zero_range = 1, with_4_days = 0;
    if (mode >= 0) calc_mode(mode, &monday_first, &zero_range, &with_4_days);
    if (monday_first) first = first == 0 ? 6 : first - 1;
    if (is_yearweek) zero_range = 0;
    int64_t contain = 7 - first;
    if (month == 1 && day <= contain && ((with_4_days && contain < 4) || (!with_4_days && first != 0))) {
        if (zero_range) { *weeks = 0; return 0; }
        (*year)--;
        doy += is_leap(*year) ? 366 : 365;
        first = (first + 53 * 7 - (is_leap(*year) ? 366 : 365)) % 7;
        contain = 7 - first;
    }
    const int64_t days = ((with_4_days && contain < 4) || (!with_4_days && first != 0)) ? doy - contain - 1 : doy - contain - 1 + 7;
    *weeks = days / 7 + 1;
    if (!zero_range && days >= 52 * 7) {
        first = (first + (is_leap(*year) ? 366 : 365)) % 7;
        if ((with_4_days && contain >= 4) || (!with_4_days && first == 0)) { (*year)++; *weeks = 1; }
    }
    return 0;
}

/* One function on an argument image of type `prim` (DATE / DATETIME / TIMESTAMP, or TIME for hour / minute / second), `prim2` /
 * `image2` for datediff's second argument.  `arg`: week / yearweek's mode (-1 = none), extract's unit (0..5 = year, month, day,
 * hour, minute, second; anything else is an unknown unit).  Returns the result as a sign- or zero-extended 64-bit value. */
int64_t bk_oracle_date_fn(const char* fn, int arg, int prim, uint64_t image, int prim2, uint64_t image2, int* is_null) {
    *is_null = 0;
    if (!strcmp(fn, "year")) return dt_year(cast_to(prim, image, P_DATETIME));                      /* :1785-1797 */
    if (!strcmp(fn, "month")) return dt_month(cast_to(prim, image, P_DATETIME));                    /* :1772-1784 */
    if (!strcmp(fn, "day") || !strcmp(fn, "dayofmonth")) return dt_day(cast_to(prim, image, P_DATETIME));   /* :1702-1714,1769-1771 */
    if (!strcmp(fn, "date")) return (int64_t)((cast_to(prim, image, P_DATETIME) >> 41) & 0x3FFFFF);  /* :1675-1687 */
    if (!strcmp(fn, "quarter")) {                                                                    /* :1432-1445 */
        const int32_t v = (int32_t)(uint32_t)cast_to(prim, image, P_DATE);
        return ((((v >> 5) & 0x1FFFF) % 13) - 1) / 3 + 1;
    }
    if (!strcmp(fn, "hour") || !strcmp(fn, "minute") || !strcmp(fn, "second")) {                  /* :1688-1701, :1410-1420, :1481-1491 */
        const int32_t t = (int32_t)(prim == P_TIME ? image : cast_to(prim, image, P_TIME));
        if (fn[0] == 'h') { int64_t a = t; if (a < 0) a = -a; return (a >> 12) & 0x3FF; }
        return fn[0] == 'm' ? (t >> 6) & 0x3F : t & 0x3F;
    }
    if (!strcmp(fn, "to_days")) return ((int64_t)cast_to(prim, image, P_TIMESTAMP) + 62167248000LL) / 86400;   /* :1572-1582 */
    if (!strcmp(fn, "to_seconds")) return (int64_t)cast_to(prim, image, P_TIMESTAMP) + 62167248000LL;        /* :1584-1594 */
    if (!strcmp(fn, "unix_timestamp")) return (int64_t)cast_to(prim, image, P_TIMESTAMP);                     /* :1315-1330 */
    if (!strcmp(fn, "datediff")) {                                                                   /* :2095-2114 */
        const int64_t t1 = (int64_t)cast_to(P_DATE, cast_to(prim, image, P_DATE), P_TIMESTAMP);
        const int64_t t2 = (int64_t)cast_to(P_DATE, cast_to(prim2, image2, P_DATE), P_TIMESTAMP);
        return (int32_t)((t1 - t2) / (3600 * 24));
    }
    if (!strcmp(fn, "extract")) {                                                                    /* :2244-2270 */
        const Civil c = localtime_fixed((int64_t)cast_to(prim, image, P_TIMESTAMP));
        switch (arg) {
            case 0: return c.year; case 1: return c.month; case 2: return c.day;
            case 3: return c.hour; case 4: return c.minute; case 5: return c.second;
            default: *is_null = 1; return 0;
        }
    }
    const uint64_t dt = cast_to(prim, image, P_DATETIME);
    const int64_t y = dt_year(dt), m = dt_month(dt), d = dt_day(dt);
    if (!strcmp(fn, "week") || !strcmp(fn, "yearweek")) {                                           /* :2027-2070 */
        int64_t year = 0, weeks = 0;
        const int yw = !strcmp(fn, "yearweek");
        if (calc_week(dt, arg, yw, &year, &weeks) != 0) { *is_null = 1; return 0; }
        return (uint32_t)(yw ? year * 100 + weeks : weeks);
    }
    if (m == 0 || d == 0 || !greg_ok(y, m, d)) { *is_null = 1; return 0; }                          /* boost::gregorian::date throws */
    if (!strcmp(fn, "dayofweek")) return day_of_week(y, m, d) + 1;                                  /* :1741-1768 */
    if (!strcmp(fn, "weekday")) { const int64_t w = day_of_week(y, m, d); return w >= 1 ? w - 1 : 6; }   /* :1875-1904 */
    if (!strcmp(fn, "dayofyear")) return day_of_year(y, m, d);                                      /* :1850-1874 */
    if (!strcmp(fn, "weekofyear")) return iso_week(y, m, d);                                        /* :2071-2093 */
    *is_null = 1;
    return 0;
}

/* the same over arrays (the GPU tests' expected columns) */
void bk_oracle_date_fn_many(const char* fn, int arg, int prim, const uint64_t* images, int prim2, const uint64_t* images2, int64_t n,
                            int64_t* out, uint8_t* is_null) {
    for (int64_t i = 0; i < n; i++) {
        int nl = 0;
        out[i] = bk_oracle_date_fn(fn, arg, prim, images[i], prim2, images2 ? images2[i] : 0, &nl);
        is_null[i] = (uint8_t)nl;
    }
}
