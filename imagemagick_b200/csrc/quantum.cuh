// quantum.cuh -- the Q16 quantum constants of the device-side colour math (QuantumRange and its reciprocal).
#pragma once

namespace mb200 {
namespace {

constexpr double QR = 65535.0;
constexpr double QS = 1.0 / 65535.0;

}  // namespace
}  // namespace mb200
