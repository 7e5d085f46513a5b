// spark_resources.hpp -- where the application tuple of the hot path comes from (SURVEY §8 row A9): the driver pod's
// annotations, parsed into the exact-int64 model of include/gangpack.h (CPU in millicores, memory in bytes, GPUs and
// executor counts in units).  Host-only, no device dependency.
//
// Reference (all under /root/reference):
//   sparkResources                        internal/extender/sparkpods.go:73-137
//   annotation keys                       internal/common/constants.go:31-50
//   resource.ParseQuantity grammar        vendor/k8s.io/apimachinery/pkg/api/resource/quantity.go:147-262 (parseQuantityString),
//                                         :264-300 (ParseQuantity), suffix.go:113-132,180-198 (suffix table / exponents)
//   Quantity.Value() (executor counts)    quantity.go:732-734 -> rounds a fractional value away from zero
//   filterToEarliestAndSort (the FIFO queue) internal/extender/sparkpods.go:54-74, internal/podspec.go:22-26
//
// A quantity the int64 model cannot hold exactly (finer than a millicore / a byte, or |v| >= 2^61) is reported as
// Unrepresentable: the embedding then lets the original Go code handle that application (INTEGRATION.md §3) -- nothing
// is rounded silently.
#pragma once

#include <algorithm>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

namespace resource {

enum class ParseStatus { Ok, ErrFormatWrong, ErrSuffix, ErrNumeric, Unrepresentable };

namespace detail {
typedef unsigned __int128 u128;
inline bool mul_overflow(u128 a, u128 b, u128* out) {
    if (a != 0 && b > (~(u128)0) / a) return true;
    *out = a * b;
    return false;
}
inline bool is_digit(char c) { return c >= '0' && c <= '9'; }

// parseQuantityString (quantity.go:147-262): sign, digits, optional ".digits", suffix.
struct Parts { bool positive = true; std::string num, denom, suffix; };
inline ParseStatus split(const std::string& str, Parts* p) {
    size_t pos = 0, end = str.size();
    if (pos < end && (str[0] == '-' || str[0] == '+')) { p->positive = str[0] != '-'; pos++; }
    while (pos < end && str[pos] == '0') pos++;                               // :163-177 leading zeros
    if (pos >= end) { p->num = "0"; return ParseStatus::Ok; }
    size_t i = pos;
    while (i < end && is_digit(str[i])) i++;                                  // :180-194 numerator
    p->num = str.substr(pos, i - pos);
    pos = i;
    if (pos >= end) { if (p->num.empty()) p->num = "0"; return ParseStatus::Ok; }
    if (p->num.empty()) p->num = "0";                                         // :197-199
    if (str[pos] == '.') {                                                    // :202-218 denominator ("1.G" is allowed, :219)
        pos++;
        i = pos;
        while (i < end && is_digit(str[i])) i++;
        p->denom = str.substr(pos, i - pos);
        pos = i;
        if (pos >= end) return ParseStatus::Ok;
    }
    const size_t suffixStart = pos;                                           // :228-238 suffix letters
    const std::string letters = "eEinumkKMGTP";
    while (pos < end && letters.find(str[pos]) != std::string::npos) pos++;
    if (pos < end && (str[pos] == '-' || str[pos] == '+')) pos++;             // :239-244 exponent sign
    while (pos < end && is_digit(str[pos])) pos++;                            // :245-256 exponent digits
    if (pos < end) return ParseStatus::ErrFormatWrong;                        // :257-260
    p->suffix = str.substr(suffixStart);
    return ParseStatus::Ok;
}

// suffixHandler.interpret (suffix.go:180-198): base 2 or 10 and the exponent.
inline ParseStatus interpret(const std::string& suf, int* base, long long* exponent) {
    static const std::map<std::string, int> dec = {{"n", -9}, {"u", -6}, {"m", -3}, {"", 0}, {"k", 3}, {"M", 6},
                                                   {"G", 9}, {"T", 12}, {"P", 15}, {"E", 18}};          // suffix.go:121-132
    static const std::map<std::string, int> bin = {{"Ki", 10}, {"Mi", 20}, {"Gi", 30}, {"Ti", 40}, {"Pi", 50}, {"Ei", 60}};  // :113-118
    auto d = dec.find(suf);
    if (d != dec.end()) { *base = 10; *exponent = d->second; return ParseStatus::Ok; }
    auto b = bin.find(suf);
    if (b != bin.end()) { *base = 2; *exponent = b->second; return ParseStatus::Ok; }
    if (suf.size() > 1 && (suf[0] == 'E' || suf[0] == 'e')) {                 // decimal exponent "e3" / "E-2"
        size_t i = 1;
        bool neg = false;
        if (suf[i] == '-' || suf[i] == '+') { neg = suf[i] == '-'; i++; }
        if (i >= suf.size()) return ParseStatus::ErrSuffix;
        long long v = 0;
        for (; i < suf.size(); ++i) {
            if (!is_digit(suf[i])) return ParseStatus::ErrSuffix;
            v = v * 10 + (suf[i] - '0');
            if (v > 1000000) return ParseStatus::ErrSuffix;                     // strconv.ParseInt would accept it, int32(parsed) would not mean it
        }
        *base = 10; *exponent = neg ? -v : v;
        return ParseStatus::Ok;
    }
    return ParseStatus::ErrSuffix;
}
}  // namespace detail

// Parse `str` like resource.ParseQuantity and return its value in units of 10^-scale (scale = 3: milli-units, 0: units),
// exactly.  roundUpFraction = true reproduces Quantity.Value() for non-integral values (away from zero) instead of
// reporting them as Unrepresentable.
inline ParseStatus ParseQuantityScaled(const std::string& str, int scale, int64_t* out, bool roundUpFraction = false) {
    using detail::u128;
    *out = 0;
    if (str.empty()) return ParseStatus::ErrFormatWrong;                       // quantity.go:265-267
    detail::Parts p;
    ParseStatus st = detail::split(str, &p);
    if (st != ParseStatus::Ok) return st;
    int base = 10; long long exponent = 0;
    st = detail::interpret(p.suffix, &base, &exponent);
    if (st != ParseStatus::Ok) return st;
    const std::string digits = p.num + p.denom;
    if (digits.size() > 36) return ParseStatus::Unrepresentable;
    u128 mant = 0;
    for (char c : digits) mant = mant * 10 + (u128)(c - '0');
    if (mant == 0) return ParseStatus::Ok;
    long long e10 = (base == 10 ? exponent : 0) - (long long)p.denom.size() + scale;
    const long long e2 = base == 2 ? exponent : 0;
    const u128 limit = (u128)1 << 61;
    if (e2 > 0 && detail::mul_overflow(mant, (u128)1 << e2, &mant)) return ParseStatus::Unrepresentable;
    bool inexact = false;
    if (e10 >= 0) {
        for (long long i = 0; i < e10; ++i) {
            if (detail::mul_overflow(mant, 10, &mant) || mant >= (limit << 8)) return ParseStatus::Unrepresentable;
        }
    } else {
        for (long long i = 0; i < -e10 && mant != 0; ++i) {
            if (mant % 10 != 0) inexact = true;
            mant /= 10;
        }
    }
    if (inexact) {
        if (!roundUpFraction) return ParseStatus::Unrepresentable;
        mant += 1;                                                              // away from zero (math.go:166-199 via Value())
    }
    if (mant >= limit) return ParseStatus::Unrepresentable;
    *out = p.positive ? (int64_t)mant : -(int64_t)mant;
    return ParseStatus::Ok;
}

}  // namespace resource

// A pod's required node affinity as the host keeps it (the device form is gangpack_host.hpp's affinity::Encoded)
namespace affinity {
struct Requirement { std::string Key, Operator; std::vector<std::string> Values; };   // v1.NodeSelectorRequirement
struct Term { std::vector<Requirement> MatchExpressions, MatchFields; };              // v1.NodeSelectorTerm
struct Program {                                   // pod.Spec.NodeSelector + RequiredDuringSchedulingIgnoredDuringExecution
    std::map<std::string, std::string> NodeSelector;
    bool HasRequired = false;                      // the required node selector is not nil
    std::vector<Term> Terms;
};
}  // namespace affinity

namespace extender {

// internal/common/constants.go:31-50
namespace common {
inline const char* const DriverCPU = "spark-driver-cpu";
inline const char* const DriverMemory = "spark-driver-mem";
inline const char* const DriverNvidiaGPUs = "spark-driver-nvidia.com/gpu";
inline const char* const ExecutorCPU = "spark-executor-cpu";
inline const char* const ExecutorMemory = "spark-executor-mem";
inline const char* const ExecutorNvidiaGPUs = "spark-executor-nvidia.com/gpu";
inline const char* const DynamicAllocationEnabled = "spark-dynamic-allocation-enabled";
inline const char* const ExecutorCount = "spark-executor-count";
inline const char* const DAMinExecutorCount = "spark-dynamic-allocation-min-executor-count";
inline const char* const DAMaxExecutorCount = "spark-dynamic-allocation-max-executor-count";
}  // namespace common

// The tuple gp_apps takes (one row), straight from the annotations.
struct ParsedSparkResources {
    int64_t DriverCPUMilli = 0, DriverMemoryBytes = 0, DriverNvidiaGPUs = 0;
    int64_t ExecutorCPUMilli = 0, ExecutorMemoryBytes = 0, ExecutorNvidiaGPUs = 0;
    int64_t MinExecutorCount = 0, MaxExecutorCount = 0;
    bool Exact = true;      // false: some quantity is outside the exact-int64 model -> the Go packer handles this application
};

// strconv.ParseBool
inline bool parseBool(const std::string& s, bool* out) {
    static const char* const t[] = {"1", "t", "T", "TRUE", "true", "True"};
    static const char* const f[] = {"0", "f", "F", "FALSE", "false", "False"};
    for (const char* x : t) if (s == x) { *out = true; return true; }
    for (const char* x : f) if (s == x) { *out = false; return true; }
    return false;
}

// sparkResources (sparkpods.go:73-137).  Returns "" on success, else the reference's error text; such drivers are skipped
// by fitEarlierDrivers (resource.go:232-237) and fail the Predicate of their own pod.
inline std::string SparkResources(const std::map<std::string, std::string>& annotations, ParsedSparkResources* out) {
    *out = ParsedSparkResources{};
    bool dynamicAllocationEnabled = false;
    auto da = annotations.find(common::DynamicAllocationEnabled);
    if (da != annotations.end() && !parseBool(da->second, &dynamicAllocationEnabled))
        return "annotation DynamicAllocationEnabled could not be parsed as a boolean";                        // :76-82
    struct Field { const char* key; int scale; int64_t* dst; bool isCount; };
    const Field fields[] = {                                                                                   // :84
        {common::DriverCPU, 3, &out->DriverCPUMilli, false},          {common::DriverMemory, 0, &out->DriverMemoryBytes, false},
        {common::DriverNvidiaGPUs, 0, &out->DriverNvidiaGPUs, false}, {common::ExecutorCPU, 3, &out->ExecutorCPUMilli, false},
        {common::ExecutorMemory, 0, &out->ExecutorMemoryBytes, false}, {common::ExecutorNvidiaGPUs, 0, &out->ExecutorNvidiaGPUs, false},
        {common::ExecutorCount, 0, nullptr, true},                    {common::DAMinExecutorCount, 0, nullptr, true},
        {common::DAMaxExecutorCount, 0, nullptr, true}};
    int64_t executorCount = 0, daMin = 0, daMax = 0;
    for (const Field& f : fields) {
        const std::string a = f.key;
        auto it = annotations.find(a);
        if (it == annotations.end()) {                                                                         // :86-99
            if (a == common::DriverNvidiaGPUs || a == common::ExecutorNvidiaGPUs) continue;
            if (!dynamicAllocationEnabled && a == common::ExecutorCount)
                return "annotation ExecutorCount is required when DynamicAllocationEnabled is false";
            if (dynamicAllocationEnabled && (a == common::DAMinExecutorCount || a == common::DAMaxExecutorCount))
                return "annotation " + a + " is required when DynamicAllocationEnabled is true";
            if (a == common::ExecutorCount || a == common::DAMinExecutorCount || a == common::DAMaxExecutorCount) continue;
            return "annotation " + a + " is missing from driver";
        }
        int64_t v = 0;
        resource::ParseStatus st = resource::ParseQuantityScaled(it->second, f.scale, &v, /*roundUpFraction=*/f.isCount);   // counts: .Value(), :108-116
        if (st == resource::ParseStatus::Unrepresentable) { out->Exact = false; continue; }
        if (st != resource::ParseStatus::Ok) return "annotation " + a + " does not have a parseable value " + it->second;   // :101-104
        if (f.dst) *f.dst = v;
        else if (a == common::ExecutorCount) executorCount = v;
        else if (a == common::DAMinExecutorCount) daMin = v;
        else daMax = v;
    }
    if (dynamicAllocationEnabled) { out->MinExecutorCount = daMin; out->MaxExecutorCount = daMax; }           // :110-115
    else { out->MinExecutorCount = executorCount; out->MaxExecutorCount = executorCount; }                    // :116-120
    return "";
}

// What ListEarlierDrivers looks at on a driver pod (sparkpods.go:45-74).
struct QueuedDriverPod {
    std::string UID;
    int64_t CreationSeconds = 0;          // CreationTimestamp
    std::string NodeName;                 // Spec.NodeName ("" = unscheduled)
    std::string SchedulerName;            // Spec.SchedulerName
    bool HasInstanceGroup = false;        // FindInstanceGroupFromPodSpec succeeded (podspec.go:29-35)
    std::string InstanceGroup;
    bool Deleting = false;                // DeletionTimestamp != nil
    affinity::Program Affinity;           // Spec.NodeSelector + the required node affinity (empty: matches every node)
};

// filterToEarliestAndSort (sparkpods.go:54-74): the drivers that must fit before `driver` may be scheduled -- unscheduled,
// same scheduler, same instance group (MatchPodInstanceGroup, podspec.go:22-26), created strictly earlier, not being
// deleted -- oldest first.  This is the order of one instance group's queue in a GP_MODE_FIFO_* batch.  (The reference
// sorts with the unstable sort.Slice; equal timestamps keep their input order here.)
inline std::vector<QueuedDriverPod> FilterToEarliestAndSort(const QueuedDriverPod& driver, const std::vector<QueuedDriverPod>& allDrivers) {
    std::vector<QueuedDriverPod> earlier;
    for (const auto& p : allDrivers) {
        if (p.NodeName.empty() && p.SchedulerName == driver.SchedulerName &&
            p.HasInstanceGroup && driver.HasInstanceGroup && p.InstanceGroup == driver.InstanceGroup &&
            p.CreationSeconds < driver.CreationSeconds && !p.Deleting)
            earlier.push_back(p);
    }
    std::stable_sort(earlier.begin(), earlier.end(),
                     [](const QueuedDriverPod& a, const QueuedDriverPod& b) { return a.CreationSeconds < b.CreationSeconds; });
    return earlier;
}

}  // namespace extender
