// datetime.h — the reference's DATE / DATETIME / TIMESTAMP / TIME images and the conversions between them, usable from host
// code (plan.cpp folds literals) and from kernels (OP_CAST on a column).
//
// Layouts (reference include/common/datetime.h:28-33,56-68; src/common/datetime.cpp:248-262):
//   DATETIME  u64  (year*13 + month) << 46 | day << 41 | hour << 36 | minute << 30 | second << 24 | microsecond
//   DATE      u32  DATETIME >> 41
//   TIMESTAMP u32  seconds since 1970-01-01 00:00:00 UTC; the reference converts in a fixed UTC+8 zone without DST
//                  (mktime_fixed_r / localtime_fixed_r, datetime.cpp:41-98, default tz_offset_hours = 8)
//   TIME      i32  sign * (hour << 12 | minute << 6 | second)
// All four order the way their images order (unsigned for the first three, signed for TIME), so comparisons and MIN/MAX work
// on the raw image; only a change of type needs the functions below (ExprValue::cast_to, include/common/expr_value.h:534-573).
// The calendar arithmetic is Richards' Julian-day-number form, checked against the oracle's restatement of the reference over
// every day of years 0..9999 and over the whole uint32 TIMESTAMP range (tests/test_datetime.py).
#pragma once
#include <stdint.h>
#include "../include/bkgpu_plan.h"

#if defined(__CUDACC__)
#define BK_HD __host__ __device__ __forceinline__
#else
#define BK_HD inline
#endif

namespace bk {

constexpr int64_t DT_ZONE_SECONDS = 8 * 3600;      // the reference's fixed zone
constexpr int64_t DT_EPOCH_JDN = 2440588;          // Julian day number of 1970-01-01

BK_HD uint64_t dt_make(uint64_t year, uint64_t month, uint64_t day, uint64_t hour, uint64_t minute, uint64_t second, uint64_t micro) {
    return ((year * 13 + month) << 46) | (day << 41) | (hour << 36) | (minute << 30) | (second << 24) | micro;
}
// days since the epoch of (year >= 0, month 1..12, day); `day` may run past the month's end, it adds linearly (as in the reference)
BK_HD int64_t dt_epoch_days(int64_t year, int64_t month, int64_t day) {
    const int64_t a = (14 - month) / 12, y = year + 4800 - a, m = month + 12 * a - 3;
    return day + (153 * m + 2) / 5 + 365 * y + y / 4 - y / 100 + y / 400 - 32045 - DT_EPOCH_JDN;
}
// DATETIME -> TIMESTAMP (datetime_to_timestamp, datetime.cpp:304-331): 0 for the zero date, a zero month or day, and anything at
// or before the epoch; the caller stores the low 32 bits (expr_value.h:551)
BK_HD int64_t dt_datetime_to_timestamp(uint64_t dt) {
    if (dt == 0) return 0;
    const int64_t ym = (int64_t)((dt >> 46) & 0x1FFFF), year = ym / 13, month = ym % 13, day = (int64_t)((dt >> 41) & 0x1F);
    if (month == 0 || day == 0) return 0;
    const int64_t t = dt_epoch_days(year, month, day) * 86400 + (int64_t)((dt >> 36) & 0x1F) * 3600 + (int64_t)((dt >> 30) & 0x3F) * 60 +
                      (int64_t)((dt >> 24) & 0x3F) - DT_ZONE_SECONDS;
    return t <= 0 ? 0 : t;
}
// TIMESTAMP -> DATETIME (timestamp_to_datetime, datetime.cpp:352-373); ts > 0 here (uint32 source), microseconds are zero
BK_HD uint64_t dt_timestamp_to_datetime(int64_t ts) {
    if (ts == 0) return 0;
    const int64_t t = ts + DT_ZONE_SECONDS;
    int64_t days = t / 86400, rem = t % 86400;
    if (rem < 0) { rem += 86400; days--; }
    const int64_t J = days + DT_EPOCH_JDN;
    const int64_t f = J + 1401 + (((4 * J + 274277) / 146097) * 3) / 4 - 38, e = 4 * f + 3, g = (e % 1461) / 4, h = 5 * g + 2;
    const int64_t day = (h % 153) / 5 + 1, month = ((h / 153 + 2) % 12) + 1, year = e / 1461 - 4716 + (14 - month) / 12;
    return dt_make((uint64_t)year, (uint64_t)month, (uint64_t)day, (uint64_t)(rem / 3600), (uint64_t)((rem % 3600) / 60), (uint64_t)(rem % 60), 0);
}
BK_HD uint64_t dt_date_to_datetime(uint64_t date) { return date << 41; }                 // datetime.h:65-67
BK_HD uint64_t dt_datetime_to_date(uint64_t dt) { return (dt >> 41) & 0x3FFFFF; }         // datetime.h:62-64
BK_HD int64_t dt_datetime_to_time(uint64_t dt) {                                          // datetime_to_time, datetime.cpp:410-419
    return (int64_t)(((dt >> 24) & 0x3F) | (((dt >> 30) & 0x3F) << 6) | (((dt >> 36) & 0x1F) << 12));
}
BK_HD bool dt_is_family(int prim) { return prim == BK_DATETIME || prim == BK_TIMESTAMP || prim == BK_DATE || prim == BK_TIME; }
// A change of type inside the family (canonical 64-bit images in and out: TIMESTAMP / DATE zero-extended, TIME sign-extended).
// TIME as the source is relative to the current date in the reference (time_to_datetime, datetime.cpp:420-442): plans that need it
// are rejected when they are compiled, so `from` is never BK_TIME here.
BK_HD uint64_t dt_family_cast(uint64_t v, int from, int to) {
    if (from == to) return v;
    const uint64_t dt = from == BK_DATETIME ? v : (from == BK_TIMESTAMP ? dt_timestamp_to_datetime((int64_t)(uint32_t)v) : dt_date_to_datetime((uint32_t)v));
    switch (to) {
        case BK_TIMESTAMP: return (uint64_t)(uint32_t)dt_datetime_to_timestamp(dt);
        case BK_DATE: return dt_datetime_to_date(dt);
        case BK_TIME: return (uint64_t)dt_datetime_to_time(dt);
        default: return dt;
    }
}

// ---- date-part and day-number functions (OP_DATEFN on the device; plan.cpp folds all-literal calls with the same code) ----
// Semantics of the reference's src/expr/internal_functions.cpp, one function at a time; result types of fn_manager.cpp:184-243.
// The argument arrives already cast to the type the reference casts it to (DateFnDef::arg_prim in plan.cpp): DATETIME for the
// field and calendar functions, DATE for quarter, TIME for hour / minute / second, TIMESTAMP for the day numbers and extract.
enum DateFn : uint8_t {
    DF_YEAR = 0, DF_MONTH, DF_DAY, DF_QUARTER, DF_HOUR, DF_MINUTE, DF_SECOND, DF_DAYOFWEEK, DF_WEEKDAY, DF_DAYOFYEAR,
    DF_WEEK, DF_YEARWEEK, DF_WEEKOFYEAR, DF_TO_DAYS, DF_TO_SECONDS, DF_UNIX_TIMESTAMP, DF_DATEDIFF, DF_EXTRACT, DF_DATE
};
enum DtUnit : uint8_t { DU_YEAR = 0, DU_MONTH, DU_DAY, DU_HOUR, DU_MINUTE, DU_SECOND };   // extract()'s units
constexpr uint64_t DT_FN_NULL = 1ull << 63;   // "the result is NULL": no date function yields this image (the largest, to_seconds, is < 2^37)
constexpr uint8_t DT_NO_MODE = 0xFF;          // week() / yearweek() called without a mode (the reference's mode -1)
constexpr int64_t DT_TO_DAYS_OFFSET = 62167248000;   // to_days / to_seconds add this to the TIMESTAMP (internal_functions.cpp:1580,1592)

// (the calendar code below is written in 32 bits: every date it sees has a year below 2^17, and the one out-of-line device function
// that runs it stays small)
BK_HD bool dt_leap(int32_t y) { return y % 4 == 0 && (y % 100 != 0 || y % 400 == 0); }
BK_HD int32_t dt_days_in_year(int32_t y) { return dt_leap(y) ? 366 : 365; }
// dt_epoch_days for years 0..131071
BK_HD int32_t dt_days32(int32_t year, int32_t month, int32_t day) {
    const int32_t a = (14 - month) / 12, y = year + 4800 - a, m = month + 12 * a - 3;
    return day + (153 * m + 2) / 5 + 365 * y + y / 4 - y / 100 + y / 400 - 32045 - (int32_t)DT_EPOCH_JDN;
}
// a date boost::gregorian::date accepts: year 1400..9999 (greg_year), month 1..12, a day inside its month.  The boost-based
// functions (dayofweek, weekday, dayofyear, week, yearweek, weekofyear) return NULL for any other.
BK_HD bool dt_gregorian_ok(int32_t y, int32_t m, int32_t d) {
    if (y < 1400 || y > 9999 || m < 1 || m > 12 || d < 1) return false;
    const int32_t last = m == 2 ? (dt_leap(y) ? 29 : 28) : (m == 4 || m == 6 || m == 9 || m == 11 ? 30 : 31);
    return d <= last;
}
// day of the week, 0 = Sunday (boost's day_of_week); 1970-01-01 was a Thursday
BK_HD int32_t dt_weekday_sun0(int32_t y, int32_t m, int32_t d) {
    const int32_t r = (dt_days32(y, m, d) + 4) % 7;
    return r < 0 ? r + 7 : r;
}
BK_HD int32_t dt_day_of_year(int32_t y, int32_t m, int32_t d) { return dt_days32(y, m, d) - dt_days32(y, 1, 1) + 1; }
// ISO 8601 week number (boost's week_number): weeks start on Monday, and a week belongs to the year that holds its Thursday
BK_HD int32_t dt_iso_week(int32_t y, int32_t m, int32_t d) {
    const int32_t day = dt_days32(y, m, d), thursday = day - (dt_weekday_sun0(y, m, d) + 6) % 7 + 3;
    const int32_t ty = thursday < dt_days32(y, 1, 1) ? y - 1 : (thursday >= dt_days32(y + 1, 1, 1) ? y + 1 : y);
    return (thursday - dt_days32(ty, 1, 1)) / 7 + 1;
}
// week() / yearweek() (calc_week and calc_mode, internal_functions.cpp:1905-2026) for a date dt_gregorian_ok accepts.  The mode's
// three flags: bit 0 = weeks start on Monday; bit 1 clear = weeks count from 0; "week 1 needs 4 days" for modes 1, 3, 4, 6.
// mode < 0 (no mode given) keeps mode 0's flags.  yearweek always counts from 1 and may move the date into the year before / after.
BK_HD void dt_calc_week(int32_t y, int32_t m, int32_t d, int mode, bool is_yearweek, int32_t& year, int32_t& week) {
    const bool monday_first = mode >= 0 && (mode & 1);
    const bool four_days = mode >= 0 && ((mode & 1) != ((mode >> 2) & 1));
    const bool zero_range = !is_yearweek && (mode < 0 || !(mode & 2));
    int32_t doy = dt_day_of_year(y, m, d), first = dt_weekday_sun0(y, 1, 1);   // weekday of January 1st
    if (monday_first) first = (first + 6) % 7;
    int32_t contain = 7 - first;                                             // days of the year in its first (partial) week
    year = y;
    if (m == 1 && d <= contain && (four_days ? contain < 4 : first != 0)) {  // the date lies before week 1
        if (zero_range) { week = 0; return; }
        year--;
        doy += dt_days_in_year(year);
        first = (first + 53 * 7 - dt_days_in_year(year)) % 7;
        contain = 7 - first;
    }
    const int32_t days = doy - contain - 1 + ((four_days ? contain < 4 : first != 0) ? 0 : 7);
    week = days / 7 + 1;
    if (!zero_range && days >= 52 * 7) {                                     // the last days may open week 1 of the next year
        first = (first + dt_days_in_year(year)) % 7;
        if (four_days ? contain >= 4 : first == 0) { year++; week = 1; }
    }
}
// localtime_fixed_r's calendar fields of a TIMESTAMP (0 included: 1970-01-01 08:00:00) as a DATETIME image
BK_HD uint64_t dt_local_fields(uint32_t ts) {
    uint32_t days = ts / 86400, rem = ts % 86400 + (uint32_t)DT_ZONE_SECONDS;
    if (rem >= 86400) { rem -= 86400; days++; }
    const int32_t J = (int32_t)days + (int32_t)DT_EPOCH_JDN;
    const int32_t f = J + 1401 + (((4 * J + 274277) / 146097) * 3) / 4 - 38, e = 4 * f + 3, g = (e % 1461) / 4, h = 5 * g + 2;
    const int32_t day = (h % 153) / 5 + 1, month = ((h / 153 + 2) % 12) + 1, year = e / 1461 - 4716 + (14 - month) / 12;
    return dt_make((uint64_t)year, (uint64_t)month, (uint64_t)day, rem / 3600, rem % 3600 / 60, rem % 60, 0);
}
// One date function on its cast argument `x` (and datediff's second argument `x2`, both as TIMESTAMP images).  `arg` is
// week / yearweek's mode (DT_NO_MODE when absent) or extract's DtUnit.  Returns the result's canonical image, or DT_FN_NULL.
BK_HD uint64_t dt_date_fn(int fn, int arg, uint64_t x, uint64_t x2) {
    const int32_t ym = (int32_t)((x >> 46) & 0x1FFFF), year = ym / 13, month = ym % 13, day = (int32_t)((x >> 41) & 0x1F);   // DATETIME fields
    switch (fn) {
        case DF_YEAR: return (uint64_t)year;                        // datetime_to_year / _month / _day: the raw fields, valid or not
        case DF_MONTH: return (uint64_t)month;
        case DF_DAY: return (uint64_t)day;
        case DF_DATE: return dt_datetime_to_date(x);
        case DF_QUARTER: {                                          // DATE image; month 0 gives (0 - 1) / 3 + 1 = 1
            const int32_t m = (((int32_t)(uint32_t)x >> 5) & 0x1FFFF) % 13;
            return (uint64_t)(int64_t)((m - 1) / 3 + 1);
        }
        case DF_HOUR: {                                             // TIME image; a negative TIME reads as its absolute value
            int64_t t = (int32_t)(uint32_t)x;
            if (t < 0) t = -t;
            return (uint64_t)((t >> 12) & 0x3FF);
        }
        case DF_MINUTE: return (uint64_t)(int64_t)(((int32_t)(uint32_t)x >> 6) & 0x3F);
        case DF_SECOND: return (uint64_t)(int64_t)((int32_t)(uint32_t)x & 0x3F);
        case DF_TO_DAYS: return (uint64_t)(((int64_t)(uint32_t)x + DT_TO_DAYS_OFFSET) / 86400);
        case DF_TO_SECONDS: return (uint64_t)((int64_t)(uint32_t)x + DT_TO_DAYS_OFFSET);
        case DF_UNIX_TIMESTAMP: return (uint64_t)(uint32_t)x;
        case DF_DATEDIFF: return (uint64_t)(int64_t)(int32_t)(((int64_t)(uint32_t)x - (int64_t)(uint32_t)x2) / 86400);
        case DF_EXTRACT: {                                          // localtime_fixed_r of the TIMESTAMP: 0 reads as 1970-01-01 08:00:00
            const uint64_t dt = dt_local_fields((uint32_t)x);
            switch (arg) {
                case DU_YEAR: return ((dt >> 46) & 0x1FFFF) / 13;
                case DU_MONTH: return ((dt >> 46) & 0x1FFFF) % 13;
                case DU_DAY: return (dt >> 41) & 0x1F;
                case DU_HOUR: return (dt >> 36) & 0x1F;
                case DU_MINUTE: return (dt >> 30) & 0x3F;
                case DU_SECOND: return (dt >> 24) & 0x3F;
                default: return DT_FN_NULL;
            }
        }
        default: break;
    }
    if (!dt_gregorian_ok(year, month, day)) return DT_FN_NULL;     // (month or day 0 included)
    switch (fn) {
        case DF_DAYOFWEEK: return (uint64_t)(dt_weekday_sun0(year, month, day) + 1);
        case DF_WEEKDAY: return (uint64_t)((dt_weekday_sun0(year, month, day) + 6) % 7);
        case DF_DAYOFYEAR: return (uint64_t)dt_day_of_year(year, month, day);
        case DF_WEEKOFYEAR: return (uint64_t)dt_iso_week(year, month, day);
        case DF_WEEK: case DF_YEARWEEK: {
            int32_t wy = 0, wk = 0;
            dt_calc_week(year, month, day, arg == DT_NO_MODE ? -1 : arg, fn == DF_YEARWEEK, wy, wk);
            return (uint64_t)(uint32_t)(fn == DF_YEARWEEK ? wy * 100 + wk : wk);
        }
        default: return DT_FN_NULL;
    }
}

}  // namespace bk
