//! DataFusion physical nodes and expressions -> the JSON operator specs of include/sailgpu.h.  NOT COMPILED here.
//!
//! Mirrors what sail_b200/plans.py writes by hand for the TPC-H plans; the expression grammar is the one documented at
//! the top of include/sailgpu.h.  Anything that has no spec returns `None`: the node stays a DataFusion node.
use std::sync::Arc;

use datafusion::arrow::datatypes::{DataType, TimeUnit};
use datafusion::logical_expr::Operator;
use datafusion::physical_expr::expressions::{BinaryExpr, CaseExpr, CastExpr, Column, InListExpr, IsNotNullExpr, IsNullExpr, LikeExpr, Literal, NegativeExpr, NotExpr};
use datafusion::physical_expr::{PhysicalExpr, ScalarFunctionExpr};
use datafusion::physical_plan::aggregates::{AggregateExec, AggregateMode};
use datafusion::physical_plan::filter::FilterExec;
use datafusion::physical_plan::joins::{HashJoinExec, NestedLoopJoinExec, PartitionMode};
use datafusion::physical_plan::projection::ProjectionExec;
use datafusion::physical_plan::repartition::RepartitionExec;
use datafusion::physical_plan::sorts::sort::SortExec;
use datafusion::physical_plan::sorts::sort_preserving_merge::SortPreservingMergeExec;
use datafusion::physical_plan::{ExecutionPlan, Partitioning};
use datafusion_common::{JoinType, ScalarValue};
use serde_json::{json, Value};

pub fn type_name(t: &DataType) -> Option<String> {
    Some(match t {
        DataType::Boolean => "Boolean".into(),
        DataType::Int8 => "Int8".into(), DataType::Int16 => "Int16".into(), DataType::Int32 => "Int32".into(), DataType::Int64 => "Int64".into(),
        DataType::UInt8 => "UInt8".into(), DataType::UInt16 => "UInt16".into(), DataType::UInt32 => "UInt32".into(), DataType::UInt64 => "UInt64".into(),
        DataType::Float32 => "Float32".into(), DataType::Float64 => "Float64".into(),
        DataType::Date32 => "Date32".into(),
        DataType::Decimal128(p, s) => format!("Decimal128({p},{s})"),
        DataType::Utf8 => "Utf8".into(), DataType::Utf8View => "Utf8View".into(),
        DataType::Timestamp(u, tz) => {
            let unit = match u { TimeUnit::Second => "s", TimeUnit::Millisecond => "ms", TimeUnit::Microsecond => "us", TimeUnit::Nanosecond => "ns" };
            match tz { Some(z) => format!("Timestamp({unit}, {z})"), None => format!("Timestamp({unit})") }
        }
        _ => return None,
    })
}

fn literal(v: &ScalarValue) -> Option<Value> {
    let t = type_name(&v.data_type())?;
    Some(match v {
        _ if v.is_null() => json!({"lit": null, "type": t}),
        ScalarValue::Boolean(Some(b)) => json!({"lit": b, "type": t}),
        ScalarValue::Int8(Some(x)) => json!({"lit": x, "type": t}), ScalarValue::Int16(Some(x)) => json!({"lit": x, "type": t}),
        ScalarValue::Int32(Some(x)) => json!({"lit": x, "type": t}), ScalarValue::Int64(Some(x)) => json!({"lit": x, "type": t}),
        ScalarValue::UInt8(Some(x)) => json!({"lit": x, "type": t}), ScalarValue::UInt16(Some(x)) => json!({"lit": x, "type": t}),
        ScalarValue::UInt32(Some(x)) => json!({"lit": x, "type": t}), ScalarValue::UInt64(Some(x)) => json!({"lit": x, "type": t}),
        ScalarValue::Float64(Some(x)) => json!({"lit": x, "type": t}),
        ScalarValue::Date32(Some(x)) => json!({"lit": x, "type": t}),
        ScalarValue::TimestampSecond(Some(x), _) | ScalarValue::TimestampMillisecond(Some(x), _)
        | ScalarValue::TimestampMicrosecond(Some(x), _) | ScalarValue::TimestampNanosecond(Some(x), _) => json!({"lit": x, "type": t}),
        ScalarValue::Decimal128(Some(x), _, _) => json!({"lit": x.to_string(), "type": t}), // unscaled integer as text (exact)
        ScalarValue::Utf8(Some(s)) | ScalarValue::Utf8View(Some(s)) => json!({"lit": s, "type": t}),
        _ => return None,
    })
}

fn op_name(op: &Operator) -> Option<&'static str> {
    Some(match op {
        Operator::Plus => "+", Operator::Minus => "-", Operator::Multiply => "*", Operator::Divide => "/", Operator::Modulo => "%",
        Operator::Eq => "=", Operator::NotEq => "!=", Operator::Lt => "<", Operator::LtEq => "<=", Operator::Gt => ">", Operator::GtEq => ">=",
        Operator::And => "and", Operator::Or => "or",
        _ => return None,
    })
}

/// `PhysicalExpr` -> expression JSON; column indices are those of the operator's input schema
pub fn expr(e: &Arc<dyn PhysicalExpr>) -> Option<Value> {
    let any = e.as_any();
    if let Some(c) = any.downcast_ref::<Column>() { return Some(json!({"col": c.index()})); }
    if let Some(l) = any.downcast_ref::<Literal>() { return literal(l.value()); }
    if let Some(b) = any.downcast_ref::<BinaryExpr>() { return Some(json!({"op": op_name(b.op())?, "l": expr(b.left())?, "r": expr(b.right())?})); }
    if let Some(n) = any.downcast_ref::<NotExpr>() { return Some(json!({"not": expr(n.arg())?})); }
    if let Some(n) = any.downcast_ref::<NegativeExpr>() { return Some(json!({"neg": expr(n.arg())?})); }
    if let Some(n) = any.downcast_ref::<IsNullExpr>() { return Some(json!({"is_null": expr(n.arg())?})); }
    if let Some(n) = any.downcast_ref::<IsNotNullExpr>() { return Some(json!({"is_not_null": expr(n.arg())?})); }
    if let Some(c) = any.downcast_ref::<CastExpr>() { return Some(json!({"cast": expr(c.expr())?, "to": type_name(c.cast_type())?})); }
    if let Some(c) = any.downcast_ref::<CaseExpr>() {
        if c.expr().is_some() { return None; } // CASE x WHEN ..: the planner has already rewritten the TPC-H shapes to searched CASE
        let arms: Option<Vec<Value>> = c.when_then_expr().iter().map(|(w, t)| Some(json!([expr(w)?, expr(t)?]))).collect();
        let els = match c.else_expr() { Some(e) => expr(e)?, None => Value::Null };
        return Some(json!({"case": arms?, "else": els}));
    }
    if let Some(l) = any.downcast_ref::<LikeExpr>() {
        if l.case_insensitive() { return None; }
        let pat = l.pattern().as_any().downcast_ref::<Literal>()?;
        let s = match pat.value() { ScalarValue::Utf8(Some(s)) | ScalarValue::Utf8View(Some(s)) => s.clone(), _ => return None };
        return Some(json!({"like": expr(l.expr())?, "pattern": s, "negated": l.negated()}));
    }
    if let Some(i) = any.downcast_ref::<InListExpr>() {
        let set: Option<Vec<Value>> = i.list().iter().map(|x| literal(x.as_any().downcast_ref::<Literal>()?.value())).collect();
        return Some(json!({"in": expr(i.expr())?, "set": set?, "negated": i.negated()}));
    }
    if let Some(f) = any.downcast_ref::<ScalarFunctionExpr>() {
        let name = f.name().to_lowercase();
        if name == "character_length" {
            // Spark's length / char_length / character_length (Utf8 or Utf8View -> Int32)
            let [arg] = f.args() else { return None };
            return Some(json!({"fn": name, "args": [expr(arg)?]}));
        }
        // date_part / date_trunc with a literal part: DataFusion's simplifier has already folded Sail's part conversion
        // (`CASE WHEN 'minute' ILIKE ..`) to a literal, as the Partial aggregate's group keys in the ClickBench snapshot show
        if name != "date_part" && name != "date_trunc" { return None; }
        let [part, arg] = f.args() else { return None };
        let part = match part.as_any().downcast_ref::<Literal>()?.value() {
            ScalarValue::Utf8(Some(s)) | ScalarValue::Utf8View(Some(s)) => s.to_lowercase(),
            _ => return None,
        };
        return Some(json!({"fn": name, "part": part, "args": [expr(arg)?]}));
    }
    None // other scalar functions (substr, ..) stay DataFusion nodes
}

pub fn filter(f: &FilterExec) -> Option<Value> {
    Some(json!({"op": "filter", "predicate": expr(f.predicate())?, "projection": f.projection()}))
}

pub fn projection(p: &ProjectionExec) -> Option<Value> {
    let exprs: Option<Vec<Value>> = p.expr().iter().map(|pe| Some(json!({"expr": expr(&pe.expr)?, "name": pe.alias}))).collect();
    Some(json!({"op": "projection", "exprs": exprs?}))
}

pub fn aggregate(a: &AggregateExec) -> Option<Value> {
    let mode = match a.mode() {
        AggregateMode::Partial => "partial", AggregateMode::Final => "final", AggregateMode::FinalPartitioned => "final_partitioned",
        AggregateMode::Single | AggregateMode::SinglePartitioned => "single",
    };
    if !a.group_expr().null_expr().is_empty() && a.group_expr().groups().len() > 1 { return None; } // grouping sets stay on the CPU
    let group_by: Option<Vec<Value>> = a.group_expr().expr().iter().map(|(e, n)| Some(json!({"expr": expr(e)?, "name": n}))).collect();
    let merging = matches!(a.mode(), AggregateMode::Final | AggregateMode::FinalPartitioned);
    let mut aggs = vec![];
    for f in a.aggr_expr() {
        if !f.order_bys().is_empty() { return None; }
        let fun = f.fun().name().to_lowercase();
        // the variance family under DataFusion's physical names (stddev / var are the sample forms); aliases stay on the CPU
        if !matches!(fun.as_str(), "sum" | "avg" | "count" | "min" | "max" | "stddev" | "stddev_pop" | "var" | "var_pop") { return None; }
        // DISTINCT over one argument of a single-mode aggregate; in a partial / final pair its state is a List column, and such
        // a pair stays a DataFusion node
        let distinct = f.is_distinct();
        let single = matches!(a.mode(), AggregateMode::Single | AggregateMode::SinglePartitioned);
        if distinct && (!single || f.expressions().len() != 1) { return None; }
        let args: Option<Vec<Value>> = f.expressions().iter().map(expr).collect();
        // input_type: type of the argument BEFORE aggregation (the final phases only see the state columns)
        let in_t = f.expressions().first().and_then(|e| e.data_type(&a.input_schema()).ok()).and_then(|t| type_name(&t));
        let mut j = json!({"fn": fun, "name": f.name(), "input_type": in_t});
        if !merging { j["args"] = Value::Array(if fun == "count" && !distinct && is_count_star(f) { vec![] } else { args? }); }
        if distinct { j["distinct"] = json!(true); }
        aggs.push(j);
    }
    Some(json!({"op": "aggregate", "mode": mode, "group_by": group_by?, "aggs": aggs}))
}

fn is_count_star(f: &datafusion::physical_expr::aggregate::AggregateFunctionExpr) -> bool {
    // count(*) arrives as count(Int64(1)) / count(Literal)
    f.expressions().iter().all(|e| e.as_any().downcast_ref::<Literal>().is_some())
}

pub fn hash_join(j: &HashJoinExec) -> Option<Value> {
    let jt = match j.join_type() {
        JoinType::Inner => "inner", JoinType::Left => "left", JoinType::Right => "right",
        JoinType::LeftSemi => "left_semi", JoinType::LeftAnti => "left_anti", JoinType::RightSemi => "right_semi", JoinType::RightAnti => "right_anti",
        _ => return None, // Full / Mark: not on the GPU path yet (sailgpu_spec_validate would refuse them as well)
    };
    let on: Option<Vec<Value>> = j.on().iter().map(|(l, r)| {
        Some(json!([l.as_any().downcast_ref::<Column>()?.index(), r.as_any().downcast_ref::<Column>()?.index()]))
    }).collect();
    let filter = match j.filter() {
        // JoinFilter expressions index an intermediate schema: column i of it is (side, index) = column_indices()[i]
        Some(f) => Some(remap_join_filter(f, j.left().schema().fields().len())?),
        None => None,
    };
    Some(json!({"op": "hash_join", "join_type": jt,
                "mode": if *j.partition_mode() == PartitionMode::CollectLeft { "collect_left" } else { "partitioned" },
                "on": on?, "filter": filter, "projection": j.projection, "null_equals_null": j.null_equality() == datafusion_common::NullEquality::NullEqualsNull}))
}

fn remap_join_filter(f: &datafusion::physical_plan::joins::utils::JoinFilter, n_left: usize) -> Option<Value> {
    use datafusion_common::JoinSide;
    fn walk(v: &mut Value, map: &[usize]) {
        match v {
            Value::Object(o) => {
                if let Some(Value::Number(i)) = o.get("col") { let k = i.as_u64().unwrap() as usize; o.insert("col".into(), json!(map[k])); return; }
                for (_, x) in o.iter_mut() { walk(x, map); }
            }
            Value::Array(a) => for x in a { walk(x, map); },
            _ => {}
        }
    }
    let map: Vec<usize> = f.column_indices().iter().map(|c| if c.side == JoinSide::Left { c.index } else { n_left + c.index }).collect();
    let mut e = expr(f.expression())?;
    walk(&mut e, &map);
    Some(e)
}

pub fn sort(s: &SortExec) -> Option<Value> {
    let keys: Option<Vec<Value>> = s.expr().iter().map(|k| {
        Some(json!({"expr": expr(&k.expr)?, "asc": !k.options.descending, "nulls_first": k.options.nulls_first}))
    }).collect();
    Some(json!({"op": "sort", "keys": keys?, "fetch": s.fetch()}))
}

/// `NestedLoopJoinExec` (inner): what DataFusion plans for scalar subqueries compared with `<` / `>` (TPC-H Q11, Q22:
/// test_tpch.plan.yaml:333,661).  The library takes the left input as the (small: at most 64 rows) build side.
pub fn nested_loop_join(j: &NestedLoopJoinExec) -> Option<Value> {
    if *j.join_type() != JoinType::Inner { return None; }
    let n_left = j.left().schema().fields().len();
    let filter = match j.filter() { Some(f) => remap_join_filter(f, n_left)?, None => Value::Null };
    let projection = j.projection.as_ref().map(|p| json!(p)).unwrap_or(Value::Null);
    Some(json!({"op": "nested_loop_join", "join_type": "inner", "filter": filter, "projection": projection}))
}

/// `SortPreservingMergeExec`: its single child has N sorted partitions; the GpuExec pushes every partition's batches as one run
/// (`"runs": "batches"`) and pulls the merged stream.
pub fn sort_preserving_merge(m: &SortPreservingMergeExec) -> Option<Value> {
    let keys: Option<Vec<Value>> = m.expr().iter().map(|k| {
        Some(json!({"expr": expr(&k.expr)?, "asc": !k.options.descending, "nulls_first": k.options.nulls_first}))
    }).collect();
    Some(json!({"op": "sort_preserving_merge", "keys": keys?, "fetch": m.fetch(), "runs": "batches"}))
}

pub fn repartition(r: &RepartitionExec) -> Option<Value> {
    match r.partitioning() {
        Partitioning::Hash(exprs, n) => {
            let e: Option<Vec<Value>> = exprs.iter().map(expr).collect();
            Some(json!({"op": "repartition", "scheme": "hash", "exprs": e?, "n": n}))
        }
        _ => None, // RoundRobinBatch re-labels whole batches: nothing to compute
    }
}

/// Dispatch on the concrete node type (same idiom as job_graph/planner.rs:179-291).
pub fn of_plan(plan: &Arc<dyn ExecutionPlan>) -> Option<Value> {
    let any = plan.as_any();
    if let Some(x) = any.downcast_ref::<FilterExec>() { return filter(x); }
    if let Some(x) = any.downcast_ref::<ProjectionExec>() { return projection(x); }
    if let Some(x) = any.downcast_ref::<AggregateExec>() { return aggregate(x); }
    if let Some(x) = any.downcast_ref::<HashJoinExec>() { return hash_join(x); }
    if let Some(x) = any.downcast_ref::<SortExec>() { return sort(x); }
    if let Some(x) = any.downcast_ref::<NestedLoopJoinExec>() { return nested_loop_join(x); }
    if let Some(x) = any.downcast_ref::<SortPreservingMergeExec>() { return sort_preserving_merge(x); }
    if let Some(x) = any.downcast_ref::<RepartitionExec>() { return repartition(x); }
    None
}
