"""trajopt_b200 — H100-native (sm_90a) batched SQP trajectory optimizer (hot path of tesseract-robotics/trajopt)."""
