// TEST INFRASTRUCTURE - CPU oracle (see oracle/model.h header).
// counted.h: an instrumented scalar for exact FLOP accounting of the hot path (BASELINE.md section 3: "algorithmic
// FLOPs per env-step = the exact count produced by the instrumented oracle").  Every arithmetic operator and math
// call on a Counted value bumps a thread-local counter: + - * / and comparisons count 1, sqrt 1, transcendental
// functions 1 each (they are O(1) in number; the count is an operation count, not a latency model).
#pragma once
#include <cmath>
#include <cstdint>
#include <limits>

namespace oracle {

struct Counted {
  double v;
  static inline thread_local uint64_t flops = 0;
  Counted() : v(0) {}
  Counted(double x) : v(x) {}
  explicit operator double() const { return v; }
  explicit operator float() const { return (float)v; }
  explicit operator int() const { return (int)v; }
  explicit operator bool() const { return v != 0; }
  Counted& operator+=(Counted o) { flops++; v += o.v; return *this; }
  Counted& operator-=(Counted o) { flops++; v -= o.v; return *this; }
  Counted& operator*=(Counted o) { flops++; v *= o.v; return *this; }
  Counted& operator/=(Counted o) { flops++; v /= o.v; return *this; }
  Counted operator-() const { return Counted(-v); }
};
#define ORACLE_BINOP(op)                                                                       \
  inline Counted operator op(Counted a, Counted b) { Counted::flops++; return Counted(a.v op b.v); } \
  inline Counted operator op(Counted a, double b) { Counted::flops++; return Counted(a.v op b); }    \
  inline Counted operator op(double a, Counted b) { Counted::flops++; return Counted(a op b.v); }    \
  inline Counted operator op(Counted a, int b) { Counted::flops++; return Counted(a.v op b); }       \
  inline Counted operator op(int a, Counted b) { Counted::flops++; return Counted(a op b.v); }
ORACLE_BINOP(+) ORACLE_BINOP(-) ORACLE_BINOP(*) ORACLE_BINOP(/)
#undef ORACLE_BINOP
#define ORACLE_CMP(op)                                                  \
  inline bool operator op(Counted a, Counted b) { return a.v op b.v; } \
  inline bool operator op(Counted a, double b) { return a.v op b; }    \
  inline bool operator op(double a, Counted b) { return a op b.v; }    \
  inline bool operator op(Counted a, int b) { return a.v op b; }       \
  inline bool operator op(int a, Counted b) { return a op b.v; }
ORACLE_CMP(<) ORACLE_CMP(>) ORACLE_CMP(<=) ORACLE_CMP(>=) ORACLE_CMP(==) ORACLE_CMP(!=)
#undef ORACLE_CMP
#define ORACLE_FN1(name) inline Counted name(Counted a) { Counted::flops++; return Counted(std::name(a.v)); }
ORACLE_FN1(sqrt) ORACLE_FN1(exp) ORACLE_FN1(expm1) ORACLE_FN1(log) ORACLE_FN1(sin) ORACLE_FN1(cos) ORACLE_FN1(cosh) ORACLE_FN1(sinh)
#undef ORACLE_FN1
inline Counted fabs(Counted a) { return Counted(std::fabs(a.v)); }
inline Counted pow(Counted a, Counted b) { Counted::flops++; return Counted(std::pow(a.v, b.v)); }
inline Counted atan2(Counted a, Counted b) { Counted::flops++; return Counted(std::atan2(a.v, b.v)); }
inline Counted fmod(Counted a, Counted b) { Counted::flops++; return Counted(std::fmod(a.v, b.v)); }

// math wrappers used by the oracle sources: std:: for float/double, the overloads above for Counted (ADL)
namespace mm {
template <class T> inline T sqrt(T x) { using std::sqrt; return sqrt(x); }
template <class T> inline T fabs(T x) { using std::fabs; return fabs(x); }
template <class T> inline T exp(T x) { using std::exp; return exp(x); }
template <class T> inline T expm1(T x) { using std::expm1; return expm1(x); }
template <class T> inline T log(T x) { using std::log; return log(x); }
template <class T> inline T sin(T x) { using std::sin; return sin(x); }
template <class T> inline T cos(T x) { using std::cos; return cos(x); }
template <class T> inline T cosh(T x) { using std::cosh; return cosh(x); }
template <class T> inline T sinh(T x) { using std::sinh; return sinh(x); }
template <class T> inline T pow(T x, T y) { using std::pow; return pow(x, y); }
template <class T> inline T atan2(T x, T y) { using std::atan2; return atan2(x, y); }
template <class T> inline T fmod(T x, T y) { using std::fmod; return fmod(x, y); }
template <class T> inline T max(T a, T b) { return a < b ? b : a; }
template <class T> inline T min(T a, T b) { return b < a ? b : a; }
inline int max(int a, int b) { return a < b ? b : a; }
inline int min(int a, int b) { return b < a ? b : a; }
template <class T> inline T eps() { return std::numeric_limits<T>::epsilon(); }
template <> inline Counted eps<Counted>() { return Counted(std::numeric_limits<double>::epsilon()); }
template <class T> inline T big() { return std::numeric_limits<T>::max(); }
template <> inline Counted big<Counted>() { return Counted(std::numeric_limits<double>::max()); }
template <class T> inline double dbl(T x) { return (double)x; }
}  // namespace mm

}  // namespace oracle
