// b2s_dates.cuh -- calendar fields of a datetime64[ns] value (DateExtractor), shared by columns_kernel (b2s_columns.cuh).
// Plain integer arithmetic: the host test suite compiles this header with a C++ compiler and compares every part with pandas.
#pragma once
#include <cstdint>

namespace b2s {

enum DatePart : int32_t {
  DP_YEAR = 0, DP_MONTH, DP_DAY, DP_HOUR, DP_MINUTE, DP_SECOND, DP_DAY_OF_WEEK, DP_DAY_OF_YEAR, DP_QUARTER,
  DP_IS_LEAP_YEAR, DP_DAYS_IN_MONTH, DP_IS_MONTH_START, DP_IS_MONTH_END, DP_IS_QUARTER_START, DP_IS_QUARTER_END,
  DP_IS_YEAR_START, DP_IS_YEAR_END, DP_WEEK,
  DP_LAST = DP_WEEK,
};

__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) {
  int64_t q = a / b;
  return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

// proleptic Gregorian calendar fields of a day count since 1970-01-01 (days-from-civil inverse)
__device__ __forceinline__ void civil_from_days(int64_t z, int& y, int& m, int& d, int& doy) {
  z += 719468;
  const int64_t era = floor_div(z, 146097);
  const int doe = (int)(z - era * 146097);                                  // [0, 146096]
  const int yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;    // [0, 399]
  const int doy_mar = doe - (365 * yoe + yoe / 4 - yoe / 100);              // [0, 365], year starting 1 March
  const int mp = (5 * doy_mar + 2) / 153;                                   // [0, 11]
  d = doy_mar - (153 * mp + 2) / 5 + 1;
  m = mp < 10 ? mp + 3 : mp - 9;
  y = (int)(yoe + era * 400) + (m <= 2 ? 1 : 0);
  const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
  const int cum[12] = {0, 31, 59, 90, 120, 151, 181, 212, 243, 273, 304, 334};
  doy = cum[m - 1] + d + ((leap && m > 2) ? 1 : 0);
}

__device__ __noinline__ int32_t date_part(int64_t ns, int part) {
  const int64_t secs = floor_div(ns, 1000000000LL);
  const int64_t days = floor_div(secs, 86400);
  const int sod = (int)(secs - days * 86400);
  switch (part) {
    case DP_HOUR: return sod / 3600;
    case DP_MINUTE: return (sod % 3600) / 60;
    case DP_SECOND: return sod % 60;
    case DP_DAY_OF_WEEK: return (int)(((days % 7) + 7 + 3) % 7);  // 1970-01-01 was a Thursday; Monday = 0
    default: break;
  }
  int y, m, d, doy;
  civil_from_days(days, y, m, d, doy);
  const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
  const int dim = (m == 2) ? (leap ? 29 : 28) : ((m == 4 || m == 6 || m == 9 || m == 11) ? 30 : 31);
  switch (part) {
    case DP_YEAR: return y;
    case DP_MONTH: return m;
    case DP_DAY: return d;
    case DP_DAY_OF_YEAR: return doy;
    case DP_QUARTER: return (m - 1) / 3 + 1;
    case DP_IS_LEAP_YEAR: return leap ? 1 : 0;
    case DP_DAYS_IN_MONTH: return dim;
    case DP_IS_MONTH_START: return d == 1;
    case DP_IS_MONTH_END: return d == dim;
    case DP_IS_QUARTER_START: return d == 1 && (m - 1) % 3 == 0;
    case DP_IS_QUARTER_END: return d == dim && m % 3 == 0;
    case DP_IS_YEAR_START: return d == 1 && m == 1;
    case DP_IS_YEAR_END: return d == 31 && m == 12;
    default: break;
  }
  // DP_WEEK: ISO 8601 week number (pd.Timestamp.week)
  const int wd = (int)(((days % 7) + 7 + 3) % 7);  // Monday = 0
  int w = (doy - wd + 9) / 7;
  auto long_year = [](int yy) {  // 53 ISO weeks: 1 January is a Thursday, or a Wednesday in a leap year
    const bool lp = (yy % 4 == 0 && yy % 100 != 0) || yy % 400 == 0;
    const int64_t yp = (int64_t)yy - 1;
    const int jan1 = (int)((yp * 365 + yp / 4 - yp / 100 + yp / 400) % 7);  // 0 = Monday (1 Jan of year 1 was a Monday)
    return jan1 == 3 || (lp && jan1 == 2);
  };
  if (w < 1) w = long_year(y - 1) ? 53 : 52;
  else if (w == 53 && !long_year(y)) w = 1;
  return w;
}

}  // namespace b2s
