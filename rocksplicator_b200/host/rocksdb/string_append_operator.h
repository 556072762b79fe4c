// rocksdb/string_append_operator.h — RocksDB's StringAppendOperator (utilities/merge_operators/string_append) and the
// MergeOperators factory that creates it.  Merge: no existing value -> the operand; otherwise existing + delim + operand.
// A delimiter of '\0' is a real byte; CreateStringAppendOperatorWithoutDelimiter() gives plain concatenation.
// GpuDB::Open recognises this class and folds its merges on the device (RSP_MERGE_STRING_APPEND); Merge below is the
// same rule for any other caller.
#pragma once
#include <memory>
#include <string>

#include "rocksdb/merge_operator.h"

namespace rocksdb {
class StringAppendOperator : public AssociativeMergeOperator {
 public:
  explicit StringAppendOperator(char delim_char) : delim_(delim_char), has_delim_(true) {}
  const char* Name() const override { return "StringAppendOperator"; }
  bool Merge(const Slice& key, const Slice* existing_value, const Slice& value, std::string* new_value,
             Logger* logger) const override {
    (void)key; (void)logger;
    if (!existing_value) {
      new_value->assign(value.data(), value.size());
      return true;
    }
    new_value->reserve(existing_value->size() + 1 + value.size());
    new_value->assign(existing_value->data(), existing_value->size());
    if (has_delim_) new_value->push_back(delim_);
    new_value->append(value.data(), value.size());
    return true;
  }
  bool has_delim() const { return has_delim_; }
  char delim() const { return delim_; }

 private:
  friend struct MergeOperators;
  StringAppendOperator() : delim_(0), has_delim_(false) {}
  char delim_;
  bool has_delim_;
};

struct MergeOperators {
  // RocksDB's default delimiter is ','
  static std::shared_ptr<MergeOperator> CreateStringAppendOperator() { return CreateStringAppendOperator(','); }
  static std::shared_ptr<MergeOperator> CreateStringAppendOperator(char delim_char) {
    return std::make_shared<StringAppendOperator>(delim_char);
  }
  // plain concatenation (the reference's SimpleMergeOperator rule), folded on the device as well
  static std::shared_ptr<MergeOperator> CreateStringAppendOperatorWithoutDelimiter() {
    return std::shared_ptr<MergeOperator>(new StringAppendOperator());
  }
};
}  // namespace rocksdb
