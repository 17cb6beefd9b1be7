// JSON -> parameter structs (model params at Init, retrieval params per request).
#pragma once
#include <string>

#include "index.h"

namespace gb {
// type: the index type the parameters are for.  The GPU_* types only record what was given here (ModelParams has_* /
// *_arg / metric_unknown); create_index checks it in their order, with their messages.
bool parse_model_params(const std::string& text, const std::string& type, ModelParams* mp, std::string* err);
bool parse_retrieval_params(const std::string& text, RetrievalParams* rp, std::string* err);
}  // namespace gb
